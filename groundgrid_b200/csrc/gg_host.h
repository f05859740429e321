// Host-only helpers (gg_host.cpp); see there for the reference citations.
#pragma once
#include <cstdint>
#include <vector>

#include "gg_internal.h"

namespace gg {
int cells_per_side(double dimension_m, float resolution);
void build_expected_points(int n, std::vector<float>& table);
void derive_geometry(double dimension_m, float resolution, unsigned flags, Const& k);

// Configuration variants of a handle.  Slots whose derived constants are identical share one variant (one
// constants record and one detect table on the device), so device memory grows with the number of distinct
// configurations in use, not with the number of slots.  Host bookkeeping only: the caller owns one device buffer
// per variant id and (re)builds it when assign() says so.  A variant no slot uses keeps its id and its buffer and is
// taken again by the next new configuration.
class ConfigRegistry {
  public:
    // every slot on variant 0 with constants k; every other variant becomes unused
    void reset(int n_slots, const CfgConst& k);
    // Points `slot` at the variant of `k` and returns its id; *build = true if that variant's device data must be
    // built first (a new id, or an unused one that held other constants).
    int assign(int slot, const CfgConst& k, bool* build);
    // Marks an unused variant's device data as unknown (a build of it failed half way): no constants match it any
    // more, so the next configuration that takes the id builds it again.
    void invalidate(int id) { vars_[id].k.reserved = 1; }   // derive_config leaves reserved at 0
    int variant_of(int slot) const { return slot_var_[slot]; }
    const CfgConst& constants(int id) const { return vars_[id].k; }
    int refs(int id) const { return vars_[id].refs; }
    int live() const;                                 // variants at least one slot uses
    int ids() const { return (int)vars_.size(); }     // variant ids handed out so far (= device buffers)

  private:
    struct Variant {
        CfgConst k;
        int refs;
    };
    std::vector<Variant> vars_;
    std::vector<int> slot_var_;
};
void move_map(double res, double& px, double& py, double nx, double ny, int& shift_i, int& shift_j);
void build_spiral_schedule(int n, std::vector<int>& level_start, std::vector<uint32_t>& visits);
void pack_cloud_range(const gg_point* src, size_t n, unsigned char* dst, size_t i0, size_t i1);
int usable_cpus();

// Tables of the skewed-layout spiral kernel (k_spiral_skew), see gg_host.cpp:build_spiral_skew.
struct SkewTables {
    bool ok = false;
    int n = 0, K = 0, KP = 0, rows = 0, levels = 0, row0 = 8;
    int lanes = 0;                       // 4 * KP
    size_t slots = 0;                    // 4 * rows * KP
    int pattern[36] = {0};               // [side][q]: slot offset of neighbour q relative to the own slot (regular visits)
    int prev_q[4] = {1, 3, 7, 5};        // neighbour index of a lane's previous cell
    std::vector<int> lane_begin, lane_end;   // [lanes] level range [begin, end) of the lane's regular run
    std::vector<int> lane_cell0;             // [lanes] cell (x + y * n) of the first regular visit; the lane then steps by +n, +1, -n, -1 (side 0..3)
    std::vector<int> cell_home;          // [n * n * 4] slots holding a copy of the cell (-1 padded; [0] first visit, [1] second visit)
    int off[4] = {0, 0, 0, 0};           // first level of ring k on side s: 3 k + off[s] (gg_internal.h:skew_regular_home)
    int home_words = 0;                  // ceil(n / 32)
    std::vector<uint32_t> home_irr;      // [n][home_words] bit per cell: its cell_home entry is not {skew_regular_home, -1, -1, -1}
    std::vector<int> irr_level_start;    // [levels + 1] CSR over levels
    std::vector<uint32_t> irr_recs;      // 16 words per irregular visit: own, nb[9], recents01, recents23, mirror, lane, cell, pad
    int max_irr_per_level = 0;
    size_t n_regular = 0, n_irregular = 0;
};
void build_spiral_skew(int n, const std::vector<int>& level_start, const std::vector<uint32_t>& visits, SkewTables& t);
bool build_spiral_records(int n, double res_sq, const std::vector<int>& level_start, const std::vector<uint32_t>& visits,
                          int dist, std::vector<uint32_t>& recs, int& max_recent);

// The spiral kernel a map of n cells per side runs, and the host tables it reads (gg_create uploads them):
//   SPIRAL_SKEW   k_spiral_skew<threads>: the skewed layout fits one CTA (4 * M lane threads + SKEW_IRR_THREADS)
//   SPIRAL_PIPE   k_spiral_pipe<threads, SPIRAL_PIPE_DIST>: at most 1024 visits per level and records that fit
//   SPIRAL_PLAIN  k_spiral: anything else
enum SpiralKind : int { SPIRAL_PLAIN = 0, SPIRAL_PIPE = 1, SPIRAL_SKEW = 2 };
struct SpiralPlan {
    SpiralKind kind = SPIRAL_PLAIN;
    int threads = 0;                     // CTA threads of the spiral launch
    int M = 0, phases = 0;               // skew: lane threads per side, rings each lane thread walks one after the other
    std::vector<int> level_start;        // the wavefront schedule (every kind; k_spiral reads it directly)
    std::vector<uint32_t> visits;
    int max_per_level = 0;
    std::vector<uint32_t> recs;          // pipe: build_spiral_records at SPIRAL_PIPE_DIST
    SkewTables skew;                     // skew: the layout (sizes, pattern, cell homes)
    std::vector<int> ph_begin, ph_end, ph_cell0;   // skew: [phase][side * M + m] (SkewView)
    std::vector<uint32_t> irr_blocks;    // skew: the irregular visits, one block of irr_chunks uint4 per level (+ 4 padding levels)
    int irr_max = 0, irr_chunks = 0;
};
void plan_spiral(int n, double res_sq, SpiralPlan& p);
}  // namespace gg

extern "C" {
// CPU-testable exports (no device needed).
int gg_host_cells_per_side(double dimension_m, float resolution);
int gg_host_expected_points(double dimension_m, float resolution, float* dst);
int gg_host_spiral_schedule(int n, int* level_start, int level_cap, uint32_t* visits, int visit_cap, int* n_levels, int* n_visits);
int gg_host_spiral_records(int n, float resolution, int dist, uint32_t* recs, int rec_cap_words, int* max_recent);
int gg_host_move_map(double res, double* pos_xy, double nx, double ny, int* shift_ij);
int gg_host_resolve_move(double res, double* pos_xy, double nx, double ny, int* shift_ij);
int gg_host_geometry_constants(double dimension_m, float resolution, unsigned flags, double* out);
int gg_host_config_constants(const gg_config* cfg, double* out);
int gg_host_config_registry(int n_slots, int n_ops, const int* op_slot, const gg_config* op_cfg, int* out);
int gg_host_pack_cloud(const gg_point* src, size_t n, unsigned char* dst);
int gg_host_packer_selftest(int threads, int n_jobs, size_t n_points, int ring_slots, int rounds, int lag);
int gg_host_spiral_plan(int n, float resolution, int* out);
int gg_host_spiral_skew(int n, int* header, int* pattern, int* lane_begin, int* lane_end, int* cell_home, int* irr_level_start, uint32_t* irr_recs, int irr_cap_words);
// homes[n * n * 4]: the slots k_detect stores each cell to (gg_internal.h:skew_home), n_table: how many cells it reads
// from the homes table; 0 when the map has no skewed layout
int gg_host_skew_homes(int n, int* homes, int* n_table);
int gg_host_decay_confidence(const gg_config* cfg, const float* occ, size_t n, float* out);
int gg_host_skew_visit_confidence(const float* d, const float* occ, size_t n, float* out);
int gg_host_outlier_walk(double dimension_m, float resolution, const double* pos_xy, const float* G, const float* C, double thr, double tol,
                         const float* origin, const float* point, long long from);
}
