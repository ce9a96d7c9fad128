// oracle/insert/lko_insert_capi.cpp — TEST INFRASTRUCTURE ONLY. The ctypes entry points of ../lko_capi.cpp (included
// unmodified, so that lko_map_insert works on the same handles as lko_create / lko_map_import / lko_map_export) plus
// lko_map_insert: the CPU restatement of lk_map_insert (include/legkilo_b200.h).
#include "../lko_capi.cpp"

namespace {

// Step 4 of KILO::predictUpdatePoint (KILO.cc:216-231) at an explicit pose: the pointWithVar of KILO.cc:125-139 /
// 219-228 for each point (float4, lidar frame), placed with rot / pos and the theta / position blocks of P, then
// UpdateVoxelMap.
void insert_at_pose(VoxelMapManager& m, const float* pts4, size_t n, const M3& rot, const V3& pos, const M3& rot_cov,
                    const M3& pos_cov) {
    std::vector<pointWithVar> pv_list(n);
    for (size_t i = 0; i < n; ++i) {
        pointWithVar& pv = pv_list[i];
        pv.point_b = vec3(pts4[4 * i], pts4[4 * i + 1], pts4[4 * i + 2]);
        pv.point_i = m.extR_ * pv.point_b + m.extT_;
        calcBodyCov(pv.point_b, m.config_setting_.dept_err_, m.config_setting_.beam_err_, pv.body_var);
        pv.point_crossmat = skew(pv.point_i);
        pv.point_w = rot * pv.point_i + pos;
        M3 rot_extR = rot * m.extR_;
        M3 rot_crossmat = rot * pv.point_crossmat;
        pv.var = (rot_extR * pv.body_var) * rot_extR.transpose() + (rot_crossmat * rot_cov) * rot_crossmat.transpose() + pos_cov;
    }
    m.UpdateVoxelMap(pv_list);
}

}  // namespace

extern "C" {

// lk_map_insert: set s = pts4[set_offsets[s] .. set_offsets[s + 1]) placed with rot[9s..], pos[3s..], rot_cov[9s..],
// pos_cov[9s..] (row-major), inserted set by set.
void lko_map_insert(void* h, uint32_t n_sets, const float* pts4, const uint32_t* set_offsets, const double* rot,
                    const double* pos, const double* rot_cov, const double* pos_cov) {
    Ctx* c = (Ctx*)h;
    for (uint32_t s = 0; s < n_sets; ++s)
        insert_at_pose(*c->map, pts4 + 4 * (size_t)set_offsets[s], set_offsets[s + 1] - set_offsets[s], to_m3(rot + 9 * (size_t)s),
                       vec3(pos[3 * s], pos[3 * s + 1], pos[3 * s + 2]), to_m3(rot_cov + 9 * (size_t)s),
                       to_m3(pos_cov + 9 * (size_t)s));
}

}  // extern "C"
