// oracle/ref_insert/ref_insert_capi.cpp — TEST INFRASTRUCTURE ONLY.
//
// The harness of ../ref/ref_capi.cpp (included unmodified, so that lkref_map_insert works on the same handles as
// lkref_create / lkref_build_voxel_map / lkref_map_export) plus lkref_map_insert: step 4 of KILO::predictUpdatePoint
// (KILO.cc:215-231) at explicit poses, built from the reference's own calcBodyCov and SKEW_SYM_MATRIX and handed to the
// reference's own VoxelMapManager::UpdateVoxelMap. Linked with the reference's unmodified sources by ./Makefile.
#include "../ref/ref_capi.cpp"

extern "C" {

// Per set, the pointWithVar of KILO.cc:125-139 / 219-228 with rot / pos / rot_cov / pos_cov in place of the filter's,
// then UpdateVoxelMap. Set s = pts4[set_offsets[s] .. set_offsets[s + 1]); 3x3 blocks row-major.
void lkref_map_insert(void* h, uint32_t n_sets, const float* pts4, const uint32_t* set_offsets, const double* rot,
                      const double* pos, const double* rot_cov, const double* pos_cov) {
    KILO& k = *((Ctx*)h)->kilo;
    for (uint32_t s = 0; s < n_sets; ++s) {
        const Mat3D R = to_m3(rot + 9 * (size_t)s), Pt = to_m3(rot_cov + 9 * (size_t)s), Pp = to_m3(pos_cov + 9 * (size_t)s);
        const Vec3D p(pos[3 * s], pos[3 * s + 1], pos[3 * s + 2]);
        std::vector<pointWithVar> pv_list(set_offsets[s + 1] - set_offsets[s]);
        for (size_t i = 0; i < pv_list.size(); ++i) {
            const float* q = pts4 + 4 * ((size_t)set_offsets[s] + i);
            pointWithVar& pv = pv_list[i];
            pv.point_b << q[0], q[1], q[2];
            pv.point_i = k.ext_rot_ * pv.point_b + k.ext_t_;
            calcBodyCov(pv.point_b, k.map_manager_->config_setting_.dept_err_, k.map_manager_->config_setting_.beam_err_,
                        pv.body_var);
            pv.point_crossmat << SKEW_SYM_MATRIX(pv.point_i);
            pv.point_w = R * pv.point_i + p;
            Mat3D rot_extR = R * k.ext_rot_;
            Mat3D rot_crossmat = R * pv.point_crossmat;
            pv.var = rot_extR * pv.body_var * rot_extR.transpose() + rot_crossmat * Pt * rot_crossmat.transpose() + Pp;
        }
        k.map_manager_->UpdateVoxelMap(pv_list);
    }
}

}  // extern "C"
