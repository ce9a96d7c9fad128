// lk_mapdev.h — host-side owner of the device map buffers (root table, node / aux / point pools,
// allocator counters) and the entry points of the map translation units.
#pragma once
#include <string>

#include "lk_device.cuh"
#include "lk_host.h"

namespace lk {

struct DevPoint;
struct FusedArgs;
struct MapDev;

class MapDevHost {
   public:
    // (Re)create an EMPTY map sized for at least these counts plus the reserve; clears the table. On failure the handle
    // holds no map (ready() is false, nothing allocated).
    int allocate(uint64_t roots, uint64_t nodes, uint64_t points, cudaStream_t s, std::string& err);
    // Make sure pools can take `extra_*` more items (grows by reallocation + copy). No-op if they fit. On failure the
    // existing pools are left as they were.
    int ensure_headroom(uint64_t extra_roots, uint64_t extra_nodes, uint64_t extra_points, cudaStream_t s,
                        std::string& err);
    void release();  // drop the map (the reserve and the tile size stay)
    MapDev dev() const;
    MapView view() const;  // what the residual path reads of dev()
    bool ready() const { return hash_cap != 0; }
    // pull the device allocator counters (free lists included) into the host mirrors
    int sync_counters(cudaStream_t s, std::string& err);
    // push the host mirrors; the free-list entries pushed since the last push become available (needs a sync_counters
    // after the last launch that freed anything)
    int push_counters(cudaStream_t s, std::string& err);
    // entries on free list l (FREE_TILES / FREE_GROUPS / FREE_SINGLES), available or pending, as of the last sync
    uint64_t free_entries(int l) const;
    uint64_t pool_bytes() const;

    // HashSlot[hash_cap] | MapNode, MapAux, HotRec[node_cap] (hot: the plane image the throughput kernel gathers) |
    // DevPoint[point_cap]
    DevBuf slots, nodes, aux, hot, points;
    // uint32_t: [0] n_nodes [1] n_roots [2] overflow [4..5] n_points (u64) [8] scratch [10..13] map_count_planes
    // [16 + 3 l .. 18 + 3 l] avail | base | top of free list l (MapDev::free_ctr)
    DevBuf counters;
    uint64_t hash_cap = 0, node_cap = 0, point_cap = 0;
    uint32_t n_roots = 0, n_nodes = 0;
    uint64_t n_points = 0;  // bump pointer (slots handed out), not the number of live points
    uint64_t reserve_roots = 0, reserve_nodes = 0, reserve_points = 0;
    uint32_t tile_slots = 52;  // the standard point tile, even_up(max_points_num + 2) (set with the map config)
    // free lists: twice as many entries as the pool holds tiles / groups / nodes, so a launch that pops and then frees
    // every object again still finds room for the pending entries
    DevBuf free_items[3];  // uint32_t
    uint64_t free_cap[3] = {0, 0, 0};
    int32_t free_avail[3] = {0, 0, 0};
    uint32_t free_base[3] = {0, 0, 0}, free_top[3] = {0, 0, 0};
    uint64_t reallocs = 0;  // pool growths since the map was created

   private:
    int size_free_lists(bool keep, cudaStream_t s, std::string& err);
};

// lk_mapbuild.cu
int map_build_device(MapDevHost& mh, const Globals& g, const float* d_xyz_world, const float* d_xyz_body, uint32_t n,
                     const double* rot, const double* rot_cov, const double* pos_cov, cudaStream_t s, std::string& err);
// cloudLidarToWorld (KILO.cc:89-106) of a raw float4 lidar cloud at pose (rot, pos): the body / world xyz map_build_device
// takes, and the world float4 (x, y, z, input w) when d_world4 is not null.
void launch_first_frame_points(const Globals& g, const float4* d_pts, uint32_t n, const double* rot, const double* pos,
                               float* d_xyz_body, float* d_xyz_world, float4* d_world4, cudaStream_t s);
// lk_insert.cu — UpdateVoxelMap (DESIGN §3.5), one per handle: shared by the streaming insert, the insert inside the
// per-scan kernel and lk_map_insert. Its scratch is stream-ordered; no call keeps its contents.
class MapInserter {
   public:
    // Before an UpdateVoxelMap of up to n points (which may create the map) in buckets of at most max_bucket points:
    // room in the pools, what earlier launches freed made available (push_counters), pending counts for every node,
    // scratch for one bucket, the touched-root counters cleared and the two-launch parity reset.
    int begin(MapDevHost& mh, const Globals& g, uint64_t n, uint32_t max_bucket, cudaStream_t s, std::string& err);
    // One bucket; returns the number of launches (0 = nothing to do). world != null: the bucket's re-projected cloud is
    // written too (the caller then skips its own re-projection kernel), and buckets of up to 4 096 points take the
    // two-launch path.
    int bucket(const MapDevHost& mh, const Globals& g, const float4* pts, const ChunkDesc* chunks, uint32_t chunk_first,
               uint32_t n_chunks, uint32_t pt_begin, uint32_t n_pts, const ScanConst* sc, const ScanStep* step,
               cudaStream_t s, float4* world = nullptr);
    // Once the stream is synchronised after the launches: report pools that ran out (push_counters clears the flag).
    int finish(const MapDevHost& mh, std::string& err) const;
    void fused_scratch(FusedArgs& fa) const;  // the scratch k_scan_fused<…, INS> inserts through
    // lk_map_insert behind its argument checks (n_sets >= 1): set t is float4 points [set_offsets[t], set_offsets[t + 1]) of
    // pts placed at (rot, pos) with the theta / position blocks (rot_cov, pos_cov), row-major 3 x 3 each. Runs in windows of
    // at most MAP_INSERT_WINDOW points, each one bucket between begin and finish, so the stream is synchronised per window.
    int insert_sets(MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
                    const double* rot, const double* pos, const double* rot_cov, const double* pos_cov, cudaStream_t s,
                    std::string& err);

   private:
    DevBuf pts_, root_, touched_, list_, counters_, pend_;  // InsertArgs; counters: [2..3] are the two-launch path's
    uint64_t pend_nodes_ = 0;  // nodes pend_ covers
    uint32_t parity_ = 0;      // the two-launch counter of the next small bucket
    // insert_sets: one window's points, its chunk table + placements (win_small_, staged in h_win_)
    DevBuf win_pts_, win_small_;
    PinnedBuf h_win_;
};
// lk_score.cu — lk_score_poses, lk_refine_poses and lk_search_poses (DESIGN §3.11-3.13), one per handle. Its scratch is
// stream-ordered; no call keeps its contents.
class PoseScorer {
   public:
    // Behind the calls' argument checks (n_poses >= 1, a map): the records of every pose of pose_set (rot / pos per pose,
    // one rot_cov / pos_cov for all), after iters refinement steps of each pose (0 = score only). Reads back the poses into
    // rot_out / pos_out and the records at them into sums_out, each when not null, in the caller's pose order. One host
    // synchronisation.
    int run(const MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
            uint32_t n_poses, const uint32_t* pose_set, const double* rot, const double* pos, const double* rot_cov,
            const double* pos_cov, int iters, double* rot_out, double* pos_out, double* sums_out, cudaStream_t s,
            std::string& err);
    // lk_search_poses behind its argument checks (n_sets >= 1, 1 <= k <= LK_SEARCH_MAX_K, every set with k to 2^32 - 1
    // candidates, a map): the candidates of each set expanded, scored and kept (best k) on the device window by window,
    // the kept ones refined, re-scored with the tight blocks and ranked. One host synchronisation.
    int search(const MapDevHost& mh, const Globals& g, uint32_t n_sets, const float* pts, const uint32_t* set_offsets,
               const uint32_t* att_offsets, const double* att_rot, const double* origin, const double* step,
               const uint32_t* counts, const double* rot_cov, const double* pos_cov, int iters, const double* rot_cov_tight,
               const double* pos_cov_tight, uint32_t k, double* rot_out, double* pos_out, double* sums_out,
               uint32_t* cand_out, cudaStream_t s, std::string& err);
    size_t device_bytes() const;  // device scratch held (both calls), lk_debug_read(h, 4, ...)
    size_t host_bytes() const;    // page-locked staging held

   private:
    // points, items | sums | ScanConst per pose (staged in h_, which also receives the read-back; search: then the ranked
    // results), the partial rows of one window, the records
    DevBuf pts_, small_, partial_, out_;
    // search: the per-set table and the attitudes; one window's candidate constants | sums | items; the running best keys
    DevBuf sets_, win_, best_;
    PinnedBuf h_;
};
// lk_mapio.cu
int map_upload_blob(MapDevHost& mh, const Globals& g, const void* blob, size_t bytes, cudaStream_t s, std::string& err);
int map_download_blob(MapDevHost& mh, void* blob, size_t capacity, size_t* bytes_out, cudaStream_t s, std::string& err);
int map_count_planes(MapDevHost& mh, uint64_t* planes, uint64_t* live_points, cudaStream_t s, std::string& err);
// drop every root whose key is outside [lo, hi] on some axis (clearMemOutOfMap, voxel_map.cc:573-594); rebuilds the table
int map_clear_outside(MapDevHost& mh, const int lo[3], const int hi[3], uint64_t* removed, cudaStream_t s, std::string& err);

}  // namespace lk
