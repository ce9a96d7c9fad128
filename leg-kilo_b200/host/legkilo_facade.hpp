// legkilo_facade.hpp — the reference's class names over the C ABI (SURVEY §8f rank 4).
//
// Header-only, needs Eigen, i.e. it is compiled INSIDE the reference's catkin workspace, not in this
// repository's build image (no Eigen / PCL / ROS here): everything below is guarded by __has_include.
// tests/test_facade_compiles.py type-checks it and instantiates its templates against a small stand-in
// for <Eigen/Dense> (tests/stubs/); the POD C ABI underneath (include/legkilo_b200.h) is what the parity
// tests cover.
//
// Mirrors: legkilo::State / ESKF (legkilo/src/core/slam/eskf.h:15-109), VoxelMapManager
// (legkilo/src/core/slam/voxel_map.h:180-244), and the per-scan entry KILO::process
// (legkilo/src/core/slam/KILO.h:28).
#pragma once
#if __has_include(<Eigen/Dense>)
#include <Eigen/Dense>

#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "legkilo_b200.h"

namespace legkilo {
namespace b200 {

using Mat3D = Eigen::Matrix3d;
using Vec3D = Eigen::Vector3d;
using StateCov = Eigen::Matrix<double, 30, 30>;
using RowMat3 = Eigen::Matrix<double, 3, 3, Eigen::RowMajor>;
using RowCov = Eigen::Matrix<double, 30, 30, Eigen::RowMajor>;

// legkilo::State <-> lk_state (rot is row-major in the ABI).
template <class StateT>
inline lk_state toAbi(const StateT& s) {
    lk_state x;
    RowMat3 R = s.rot_;
    std::memcpy(x.rot, R.data(), sizeof(x.rot));
    const Vec3D* v[9] = {&s.pos_, &s.vel_, &s.ba_, &s.bw_, &s.grav_, &s.imu_a_, &s.imu_w_, &s.bv_, &s.contact_};
    double* d[9] = {x.pos, x.vel, x.ba, x.bw, x.grav, x.imu_a, x.imu_w, x.bv, x.contact};
    for (int i = 0; i < 9; ++i) std::memcpy(d[i], v[i]->data(), 24);
    return x;
}
template <class StateT>
inline void fromAbi(const lk_state& x, StateT& s) {
    s.rot_ = Eigen::Map<const RowMat3>(x.rot);
    Vec3D* v[9] = {&s.pos_, &s.vel_, &s.ba_, &s.bw_, &s.grav_, &s.imu_a_, &s.imu_w_, &s.bv_, &s.contact_};
    const double* d[9] = {x.pos, x.vel, x.ba, x.bw, x.grav, x.imu_a, x.imu_w, x.bv, x.contact};
    for (int i = 0; i < 9; ++i) *v[i] = Eigen::Map<const Vec3D>(d[i]);
}

// Owns the device context; what KILO keeps instead of unique_ptr<ESKF> + unique_ptr<VoxelMapManager>.
class Core {
   public:
    template <class EskfConfig, class VoxelMapConfig>
    Core(const EskfConfig& ec, const VoxelMapConfig& mc, const Mat3D& ext_rot, const Vec3D& ext_t, int device = 0) {
        static_assert(sizeof(EskfConfig) == sizeof(lk_eskf_cfg), "ESKF::Config layout (eskf.h:49-65)");
        std::memcpy(&ec_, &ec, sizeof(ec_));
        lk_map_cfg m{};
        m.max_voxel_size = mc.max_voxel_size_; m.planner_threshold = mc.planner_threshold_; m.beam_err = mc.beam_err_;
        m.dept_err = mc.dept_err_; m.sigma_num = mc.sigma_num_; m.max_layer = mc.max_layer_; m.max_points_num = mc.max_points_num_;
        for (int i = 0; i < 5 && i < (int)mc.layer_init_num_.size(); ++i) m.layer_init_num[i] = mc.layer_init_num_[i];
        RowMat3 Re = ext_rot;
        if (lk_create(&ec_, &m, Re.data(), ext_t.data(), device, &h_) != LK_OK) throw std::runtime_error(lk_last_error(nullptr));
        Q_.resize(900);
        lk_init_process_cov(&ec_, Q_.data());  // ESKF::initProcessCovQ (eskf.cc:47-62)
    }
    ~Core() { lk_destroy(h_); }
    Core(const Core&) = delete;
    Core& operator=(const Core&) = delete;

    // VoxelMapManager::BuildVoxelMap (voxel_map.cc:287-334). xyz arrays: n x 3 floats.
    void BuildVoxelMap(const float* xyz_world, const float* xyz_body, size_t n, const Mat3D& rot, const Mat3D& rot_cov,
                       const Mat3D& pos_cov) {
        RowMat3 R = rot, Cr = rot_cov, Cp = pos_cov;
        check(lk_map_build(h_, xyz_world, xyz_body, n, R.data(), Cr.data(), Cp.data()));
    }

    // The first-frame branch of KILO::process (KILO.cc:331-353): StateInitial over the frame's inertial queue (exactly one of
    // imu / kin non-empty), cloudLidarToWorld at the state's position and BuildVoxelMap, in one call. xyzw: the raw cloud as
    // float4 (x, y, z, w), as lk_decode_pointcloud2 writes it; world_xyzw (optional) receives cloud_down_world_out.
    // Returns false with nothing changed when the cloud or the queue is empty ("Data packet is not ready", KILO.cc:326-329).
    template <class StateT>
    bool firstFrame(StateT& state, StateCov& cov, double& last_predict_time, double& last_update_time, double& acc_norm,
                    const std::vector<float>& xyzw, double end_time, const std::vector<lk_imu_meas>& imu,
                    const std::vector<lk_kinimu_meas>& kin, double gravity, std::vector<float>* world_xyzw = nullptr) {
        lk_state x = toAbi(state);
        RowCov P;
        lk_stream_clock clk{};
        double an = 0.0;
        if (world_xyzw) world_xyzw->resize(xyzw.size());
        const int rc = lk_first_frame(h_, &x, P.data(), &clk, &an, xyzw.data(), (uint32_t)(xyzw.size() / 4), end_time,
                                      imu.empty() ? nullptr : imu.data(), kin.empty() ? nullptr : kin.data(),
                                      (uint32_t)(imu.empty() ? kin.size() : imu.size()), gravity,
                                      world_xyzw ? world_xyzw->data() : nullptr);
        if (rc == LK_ERR_NOT_READY) return false;
        check(rc);
        fromAbi(x, state);
        cov = P;
        last_predict_time = clk.last_predict_time;
        last_update_time = clk.last_update_time;
        acc_norm = an;  // acc_norm_ (KILO.cc:349)
        return true;
    }

    // The second lambda of KILO::process (KILO.cc:367-396) for one scan whose points are already in the
    // canonical (stable, ascending curvature) order. Exactly one of imu / kin may be non-empty.
    template <class StateT>
    size_t processScan(StateT& state, StateCov& cov, double& last_predict_time, double& last_update_time,
                       const std::vector<float>& xyzt, const std::vector<uint32_t>& bucket_offsets,
                       const std::vector<double>& bucket_times, std::vector<lk_imu_meas>& imu, std::vector<lk_kinimu_meas>& kin,
                       double gravity, double acc_norm, std::vector<float>& world_xyzi, int iters = 1, bool update_map = true) {
        lk_state x = toAbi(state);
        RowCov P = cov;
        lk_stream_clock clk{last_predict_time, last_update_time};
        uint32_t n_eff = 0, used = 0;
        const uint32_t n = (uint32_t)(xyzt.size() / 4);
        world_xyzi.resize(xyzt.size());
        check(lk_process_scan(h_, &x, P.data(), Q_.data(), &clk, xyzt.data(), n, bucket_offsets.data(), bucket_times.data(),
                              (uint32_t)bucket_times.size(), imu.empty() ? nullptr : imu.data(), kin.empty() ? nullptr : kin.data(),
                              (uint32_t)(imu.empty() ? kin.size() : imu.size()), gravity, acc_norm, iters, update_map ? 1 : 0,
                              world_xyzi.data(), &n_eff, &used));
        fromAbi(x, state);
        cov = P;
        last_predict_time = clk.last_predict_time;
        last_update_time = clk.last_update_time;
        if (!imu.empty()) imu.erase(imu.begin(), imu.begin() + used);  // the deque pop_front of KILO.cc:382, :388
        if (!kin.empty()) kin.erase(kin.begin(), kin.begin() + used);
        return n_eff;  // success_pts_size_out
    }

    // lk_score_poses: the sums the LiDAR update would form at each candidate pose, against the map, with no filter, map or
    // staged batch touched. xyzw: float4 lidar-frame points, set s = points [set_offsets[s], set_offsets[s+1]); pose m places
    // set pose_set[m] at (rot[m], pos[m]); rot_cov / pos_cov: the theta / position blocks of P shared by every pose.
    // Returns LK_SCORE_STRIDE doubles per pose, laid out as LK_SCORE_* (count at LK_SCORE_COUNT).
    std::vector<double> scorePoses(const std::vector<float>& xyzw, const std::vector<uint32_t>& set_offsets,
                                   const std::vector<uint32_t>& pose_set, const std::vector<Mat3D>& rot,
                                   const std::vector<Vec3D>& pos, const Mat3D& rot_cov, const Mat3D& pos_cov) {
        const size_t n = pose_set.size();
        if (rot.size() != n || pos.size() != n || set_offsets.empty())
            throw std::invalid_argument("scorePoses: one rot / pos per pose, and set_offsets of n_sets + 1 entries");
        std::vector<double> R(9 * n), p(3 * n), out(LK_SCORE_STRIDE * n);
        for (size_t m = 0; m < n; ++m) {
            RowMat3 Rm = rot[m];
            std::memcpy(&R[9 * m], Rm.data(), 72);
            std::memcpy(&p[3 * m], pos[m].data(), 24);
        }
        RowMat3 Cr = rot_cov, Cp = pos_cov;
        check(lk_score_poses(h_, (uint32_t)(set_offsets.size() - 1), xyzw.data(), set_offsets.data(), (uint32_t)n,
                             pose_set.data(), R.data(), p.data(), Cr.data(), Cp.data(), out.data()));
        return out;
    }

    // lk_refine_poses: each candidate pose refined in place by `iters` steps of the LiDAR update with the theta / position
    // blocks of P held at rot_cov / pos_cov, against the map, with no filter, map or staged batch touched. Inputs as
    // scorePoses. Returns the records at the refined poses (LK_SCORE_STRIDE doubles per pose, laid out as LK_SCORE_*).
    std::vector<double> refinePoses(const std::vector<float>& xyzw, const std::vector<uint32_t>& set_offsets,
                                    const std::vector<uint32_t>& pose_set, std::vector<Mat3D>& rot, std::vector<Vec3D>& pos,
                                    const Mat3D& rot_cov, const Mat3D& pos_cov, int iters) {
        const size_t n = pose_set.size();
        if (rot.size() != n || pos.size() != n || set_offsets.empty())
            throw std::invalid_argument("refinePoses: one rot / pos per pose, and set_offsets of n_sets + 1 entries");
        std::vector<double> R(9 * n), p(3 * n), out(LK_SCORE_STRIDE * n);
        for (size_t m = 0; m < n; ++m) {
            RowMat3 Rm = rot[m];
            std::memcpy(&R[9 * m], Rm.data(), 72);
            std::memcpy(&p[3 * m], pos[m].data(), 24);
        }
        RowMat3 Cr = rot_cov, Cp = pos_cov;
        check(lk_refine_poses(h_, (uint32_t)(set_offsets.size() - 1), xyzw.data(), set_offsets.data(), (uint32_t)n,
                              pose_set.data(), R.data(), p.data(), Cr.data(), Cp.data(), iters, R.data(), p.data(),
                              out.data()));
        for (size_t m = 0; m < n; ++m) {
            rot[m] = Eigen::Map<const RowMat3>(&R[9 * m]);
            pos[m] = Eigen::Map<const Vec3D>(&p[3 * m]);
        }
        return out;
    }

    // lk_search_poses: per set, its attitudes (att_offsets) times one position lattice (counts, step, origin[s]) scored
    // with rot_cov / pos_cov, the best k kept, refined by `iters` steps, re-scored with the tight blocks and ordered by the
    // tight count, on the device. xyzw / set_offsets as scorePoses. rot / pos receive the k results of each set (entry
    // s k + j), cand their candidate indices; returns their tight records (LK_SCORE_STRIDE doubles each, laid out as
    // LK_SCORE_*).
    std::vector<double> searchPoses(const std::vector<float>& xyzw, const std::vector<uint32_t>& set_offsets,
                                    const std::vector<uint32_t>& att_offsets, const std::vector<Mat3D>& att,
                                    const std::vector<Vec3D>& origin, const Vec3D& step, const uint32_t counts[3],
                                    const Mat3D& rot_cov, const Mat3D& pos_cov, int iters, const Mat3D& rot_cov_tight,
                                    const Mat3D& pos_cov_tight, uint32_t k, std::vector<Mat3D>& rot, std::vector<Vec3D>& pos,
                                    std::vector<uint32_t>& cand) {
        if (set_offsets.empty() || att_offsets.size() != set_offsets.size() || origin.size() + 1 != set_offsets.size() ||
            att.size() < att_offsets.back())
            throw std::invalid_argument("searchPoses: set_offsets / att_offsets of n_sets + 1 entries, one origin per set");
        const size_t n_sets = origin.size(), n = n_sets * k;
        std::vector<double> A(9 * att.size()), O(3 * n_sets), R(9 * n), p(3 * n), out(LK_SCORE_STRIDE * n);
        for (size_t a = 0; a < att.size(); ++a) {
            RowMat3 Ra = att[a];
            std::memcpy(&A[9 * a], Ra.data(), 72);
        }
        for (size_t s = 0; s < n_sets; ++s) std::memcpy(&O[3 * s], origin[s].data(), 24);
        RowMat3 Cr = rot_cov, Cp = pos_cov, Crt = rot_cov_tight, Cpt = pos_cov_tight;
        cand.resize(n);
        check(lk_search_poses(h_, (uint32_t)n_sets, xyzw.data(), set_offsets.data(), att_offsets.data(), A.data(), O.data(),
                              step.data(), counts, Cr.data(), Cp.data(), iters, Crt.data(), Cpt.data(), k, R.data(), p.data(),
                              out.data(), cand.data()));
        rot.resize(n);
        pos.resize(n);
        for (size_t m = 0; m < n; ++m) {
            rot[m] = Eigen::Map<const RowMat3>(&R[9 * m]);
            pos[m] = Eigen::Map<const Vec3D>(&p[3 * m]);
        }
        return out;
    }

    // VoxelMapManager::mapSliding (voxel_map.cc:552-571): drop the root voxels that left the +-half_map_size window.
    bool mapSliding(const Vec3D& position_last, uint64_t* removed = nullptr) {
        int32_t slid = 0;
        check(lk_map_slide(h_, position_last.data(), &slid, removed));
        return slid != 0;
    }

    // TrajectorySaver::write (trajectory_saver.hpp:43-50): one TUM line of the current pose.
    template <class StateT>
    std::string tumLine(double timestamp, const StateT& state) const {
        RowMat3 R = state.rot_;
        char buf[256];
        const int n = lk_tum_line(timestamp, R.data(), state.pos_.data(), buf, sizeof(buf));
        if (n < 0) throw std::runtime_error("lk_tum_line");
        return std::string(buf, (size_t)n);
    }

    lk_handle handle() const { return h_; }

   private:
    void check(int rc) const {
        if (rc != LK_OK) throw std::runtime_error(lk_last_error(h_));
    }
    lk_handle h_ = nullptr;
    lk_eskf_cfg ec_{};
    std::vector<double> Q_;
};

}  // namespace b200
}  // namespace legkilo
#endif  // __has_include(<Eigen/Dense>)
