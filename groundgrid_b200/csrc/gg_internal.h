// Internal definitions shared by the kernels (gg_kernels.cu) and the C-ABI (gg_capi.cu).
// Not installed; the public boundary is include/groundgrid_b200.h.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cfloat>

#include "groundgrid_b200.h"

namespace gg {

// ---- device layer slots (per map slot, each N*N floats, column-major) -------------------
// "ground" and "groundpatch" come first and are contiguous: they are the rolling terrain
// prior, the only state that survives a scan (SURVEY.md section 0) and what NCCL broadcasts.
enum Layer : int {
    L_GROUND = 0,       // "ground"            terrain height G
    L_GROUNDPATCH = 1,  // "groundpatch"       confidence C
    L_OBSTACLES = 2,    // "points" after labelling: non-ground points per cell (GroundSegmentation.cpp:147,176)
    L_VARIANCE = 3,     // "variance"          m2 / (count + FLT_MIN)            (:323)
    L_MINH = 4,         // "minGroundHeight"
    L_COUNT = 5,        // "points" during rasterisation: kept points per cell   (:309)
    L_MAXH = 6,         // "maxGroundHeight"   (dead layer)
    L_GCAND = 7,        // "groundCandidates"  (dead layer)
    L_PLANEDIST = 8,    // "planeDist"         (dead layer)
    L_M2 = 9,           // "m2"
    L_MEAN = 10,        // "meanVariance"      Welford mean
    L_RAW = 11,         // "pointsRaw"         (dead layer)
    L_NUM = 12,
    L_NUM_LIVE = 6,     // layers [0, 6) exist always; [6, 12) only with GG_FLAG_FULL_LAYERS
};

// per-point class codes (upper byte of PointAux code)
enum PointClass : unsigned {
    PC_ABSENT = 0,          // outside the map / NaN: never part of the output cloud
    PC_KEPT = 1,            // rasterised, labelled by the height test
    PC_KEPT_BORDER = 2,     // rasterised, but cell index >= N-3: vanishes from the output (:167-168)
    PC_IGNORED = 3,         // ring > max_ring or closer than sqrt(12) m: labelled, not rasterised (:237-240)
    PC_IGNORED_BORDER = 4,  // ignored and in a border cell: vanishes
    PC_OUTLIER = 5,         // below-ground outlier: always labelled ground (:270,185-189)
};

// Geometry constants of a handle (grid_map::GridMap::setGeometry), derived once in gg_create on the host.
struct Const {
    int N, N2;
    int full_layers;
    float res_f;            // (float) map.getResolution()
    double res;             // map.getResolution()  == (double) res_f
    double rres;            // 1 / res (only to skip IEEE divisions whose integer part is not in doubt)
    double len, half;       // N * res, 0.5 * len
    double res_sq;          // res * res  (std::pow(resolution, 2.0), :332,356,463)
};

// Constants derived from one configuration on the host, with the reference's own expressions (so the fp64 values
// are what the reference's compiler computes).  One record per configuration variant (gg_host.h:ConfigRegistry); it
// travels by value in the SlotParams of every scan.  No padding: records are compared bytewise.
struct CfgConst {
    int max_ring;
    float pc_var_thresh_f;  // (float) point_count_cell_variance_threshold (float >= int compare, :374)
    double min_outlier_conf, outlier_tol;
    double gp_thresh;       // ground_patch_detection_minimum_point_count_threshold
    double df_sq, mdf_sq, mdf10_sq, psc_sq;
    double occ_factor, occ_factor2, dec_factor;
    double lab_fac, lab_thres, lab_obs;
    int decay_floor_ok;     // decay of a confidence <= 0.001f gives 0.001f again (checked on the host for dec_factor)
    int reserved;           // zero
};
static_assert(sizeof(CfgConst) == 120, "CfgConst has no padding");

// Per-scan, per-slot parameters (changes every scan / pose update).
struct SlotParams {
    // configuration variant of the slot (set by every launch that reads it; zero otherwise): its constants by value
    // (a pointer would add a dependent load to the start of every block) and its detect table, [N2] per-cell constants
    // of the patch detection (gg_kernels.cu:k_build_detect_table), built once and immutable while a slot uses it
    CfgConst cfg;
    const float4* detect_tab;
    double px, py;        // map centre position
    double t20, t21, t22, t23;  // row 2 of T_base_from_map (seed of exposed cells)
    float ox, oy, oz;     // cloud origin
    float base_z_f;       // (float) base_z
    int n_points;
    int shift_i, shift_j; // pending roll (index shift): new(r,c) = old(r + shift_i, c + shift_j)
    int slot;
    const gg_point* src;  // device pointer of this scan's cloud (the slot's own buffer or a caller-owned one)
    // packed cloud (host-side packing of the batched host-buffer path): x | y | z as float[n_pad]
    // followed by ring as uint16[n_pad], n_pad = n_points rounded up to 8; null -> `src` is used
    const float* packed;
    // batched calls on a list of slots: the scan's position in the call (where its part of the caller's buffer starts)
    // and the layer "points" names for the slot (LAYER_POINTS); appended, so the fields above keep their offsets
    int pos;
    int points_layer;
    // a scan of GG_SCAN_DEVICE_MASK whose slot's stored mask is 0 (set by k_stage_poses, with n_points 0): every kernel
    // of the scan returns at entry for it; appended, so the fields above keep their offsets
    int skip;
};

// Per-scan destinations of the output kernels (launch_output).  They sit in the staging entry next to the scans'
// SlotParams, in a parallel array with the same index: the handle's own buffers for gg_get_output, the caller's for
// gg_run_scans_to_device.
struct OutDest {
    uint8_t* labels;   // [n_points] copy of the scan's labels; null: none
    uint32_t* index;   // input index of each selected output point; null: none
    gg_point* cloud;   // the selected output points (intensity = label); null: none
    int* count;        // receives the number of selected points; null: none
    unsigned select;   // GG_SELECT_* bits: labels that enter index / cloud / count
    int reserved;      // zero
};

// Spiral kernels (the path is chosen by gg_host.cpp:plan_spiral)
constexpr int SPIRAL_THREADS = 512;   // CTA threads of the plain k_spiral
constexpr int SPIRAL_PIPE_DIST = 2;   // prefetch distance (levels) of k_spiral_pipe, and of the records built for it
constexpr int SKEW_IRR_THREADS = 64;  // threads of k_spiral_skew that run the irregular visits (after the 4 * M lane threads)
constexpr int SKEW_XCH_DEPTH = 2;     // levels in the exchange ring of k_spiral_skew: a value written at level l is read at l + 1

// Device side of the skewed-layout spiral (gg_host.h:SkewTables); null sk -> not used.
struct SkewView {
    float2* sk;             // [n_slots][slots] (G, C) in (side, level, ring) order
    float* sd;              // [n_slots][slots] decayed confidence the visit will store, -1: confidence unchanged
    size_t slots;
    const int* cell_home;   // [N2][4]
    // Lane threads are time-shared: ring k and ring k + M of one side are never active at the same
    // level (ring k spans levels ~[3k, 5k]), so thread (side, m) walks rings m, m + M, m + 2M ... one
    // after the other ("phases").  [phase][side * M + m] tables; an empty phase has begin == end.
    const int* ph_begin;    // level range [begin, end) of the regular run
    const int* ph_end;
    const int* ph_cell0;    // cell (x + y * N) of the first regular visit
    int M, phases;
    // irregular visits, one fixed-size block per level (irr_chunks x uint4):
    //   words [ (v * 9 + q) * 2 + {0, 1} ] = slot of neighbour q of visit v, producer lane if it was
    //                                        written one level ago (else 0xffffffff)
    //   words [ irr_max * 18 + v * 4 + {0..3} ] = own slot (0xffffffff: no visit), mirror slot, lane, cell
    const uint4* irr_blocks;
    int irr_max, irr_chunks;
    int KP, rows, row0, lanes, levels;
    int pattern[36];
    // Homes of the cells (skew_home): bit x % 32 of home_irr[y * home_words + x / 32] is set for a cell whose homes in
    // cell_home are not the single slot skew_regular_home derives (ring corners, lane ends, the centre, the border)
    const uint32_t* home_irr;   // [N][home_words]
    int home_words;             // ceil(N / 32)
    int K;                      // rings 0 .. K - 1 are swept, ring K is the border they read
    int off[4];                 // first level of ring k on side s: 3 k + off[s]
};

// The slot cell (x, y) of an n x n map would take in the skewed layout if its lane visited it once, one level per cell
// (gg_host.cpp:build_spiral_skew): ring k = Chebyshev distance from the centre cell c minus one, side and position j along
// the side as the sequential sweep walks them, level 3 k + off[side] + j.  -1 outside rings 0 .. K.
__host__ __device__ __forceinline__ int skew_regular_home(int n, int K, int KP, int rows, int row0, const int* off, int x, int y) {
    const int c = n / 2 - 1;
    const int ax = x > c ? x - c : c - x, ay = y > c ? y - c : c - y;
    const int k = (ax > ay ? ax : ay) - 1;
    if (k < 0 || k > K) return -1;
    const int p = c - 1 - k, q = c + 1 + k;
    int s, j;
    if (x == p && y < q) {
        s = 0;   // (p, p + j)
        j = y - p;
    } else if (y == p && x < q) {
        s = 1;   // (p + j, p)
        j = x - p;
    } else if (x == q) {
        s = 2;   // (q, q - j)
        j = q - y;
    } else {
        s = 3;   // (q - j, q)
        j = q - x;
    }
    return (s * rows + 3 * k + off[s] + j + row0) * KP + k + 1;
}

// The homes of cell (x, y) of an n x n map: what cell_home holds for it (-1 padded), read from there only for the cells
// home_irr marks.  k_detect stores every cell through it; gg_host_skew_homes runs it on the host.
__host__ __device__ __forceinline__ int4 skew_home(const SkewView& w, int n, int x, int y) {
    if ((w.home_irr[y * w.home_words + (x >> 5)] >> (x & 31)) & 1u) {
#ifdef __CUDA_ARCH__
        return __ldg(reinterpret_cast<const int4*>(w.cell_home) + x + y * n);
#else
        const int* h = w.cell_home + 4 * ((size_t)x + (size_t)y * n);
        return make_int4(h[0], h[1], h[2], h[3]);
#endif
    }
    return make_int4(skew_regular_home(n, w.K, w.KP, w.rows, w.row0, w.off, x, y), -1, -1, -1);
}

// Pointers / strides of the handle's device arena, passed to kernels by value.
struct View {
    Const k;
    float* layers;        // [n_slots][n_layers][N2]
    int n_layers;
    const float* expected;  // [N2] expectedPoints table (GroundSegmentation.cpp:40-46)
    gg_point* points;     // [n_slots][pcap]
    unsigned char* packed;  // [n_slots][14 * pcap] packed clouds (allocated on first use)
    uint2* zw;            // [n_slots][pcap] per input point: (z bits, position in the cell's segment | run-head flag << 31)
    uint32_t* runj;       // [n_slots][pcap] run heads only: arrival number of the run in its cell | (run length - 1) << 26
    float* zsorted;       // [n_slots][pcap] z of kept points grouped by cell: the cell's segment is a sequence of runs
    uint2* rundir;        // [n_slots][pcap] run directory, cell by cell at cellstart: (run id = point index >> 5, first position | (length - 1) << 26)
    float* dist;          // [n_slots][pcap] hypotf(x - ox, y - oy)
    uint32_t* code;       // [n_slots][pcap] class << 24 | cell
    uint8_t* labels;      // [n_slots][pcap]
    unsigned long long* cnt64;  // [n_slots][N2] runs of the cell << 32 | kept points of the cell (one atomic per run)
    int* raw_i;           // [n_slots][N2] inside points per cell (full layers)
    int* cellstart;       // [n_slots][N2] exclusive scan of the per-cell point counts
    int4* worklist;       // [n_slots][N2] non-empty cells grouped by count class, heaviest first: (cell, points, runs, segment start)
    int* wl_count;        // [n_slots][2] entries of the worklist, kept points of the scan
    int* cell_agg;        // [n_slots][cell_tiles][65] per tile of 4096 cells: cells per count class, kept points
    int cell_tiles;       // ceil(N2 / 4096)
    uint32_t* out_index;  // [n_slots][pcap]
    int* out_counts;      // [n_slots][3 * out_blocks + 1]  (+1: n_out)
    gg_point* out_cloud;  // [n_slots][pcap] (allocated lazily)
    float* roll_scratch;  // [n_slots][2][N2]
    size_t pcap;
    int out_blocks;       // ceil(pcap / OUT_TILE)
    // spiral wavefront schedule (shared by all slots)
    const int* level_start;   // [levels + 1]
    const uint32_t* visits;   // [n_visits]  x | y << 16
    int levels;
    // pipelined spiral (k_spiral_pipe): 16-byte records, see gg_host.cpp:build_spiral_records
    const uint4* spiral_recs; // null -> plain k_spiral
    int spiral_threads;       // CTA threads of the spiral launch (gg_host.h:SpiralPlan::threads)
    SkewView skew;            // skew.sk != null -> k_skew + k_spiral_skew + k_unskew replace k_spiral_pipe

    __host__ __device__ float* layer(int slot, int l) const { return layers + ((size_t)slot * n_layers + l) * k.N2; }
};

constexpr int RASTER_TILE = 2048;
constexpr int RASTER_THREADS = 256;
constexpr int OUT_TILE = 1024;

// kernels of the pipeline, as reported by the profiling hooks (gg_profile_read)
enum KernelId : int {
    K_RASTERIZE = 0, K_CELL_TILES, K_CELL_PLACE, K_SCATTER, K_CELL_STATS, K_DETECT, K_SPIRAL, K_LABEL, K_ROLL_GATHER, K_ROLL_COMMIT, K_OUT_COUNT, K_OUT_SCAN,
    K_OUT_WRITE, K_UNPACK, K_TERRAIN, K_EVAL, K_LAYER_COPY, K_LAYER_RANGE, K_LAYER_IMAGE, K_SAMPLE, K_POINT_INFO, K_STAGE_POSES, K_POSE_RESOLVE,
    K_STORE_COUNTS, K_RESET_MAPS, K_STAGE_PARTS, K_STORE_PART_COUNTS, K_STORE_CONFIGS, K_REBUILD_DETECT, K_RESTORE_MAPS, K_SAVE_MAPS,
    K_NUM
};

// Optional per-kernel CUDA-event timing (bench.py's roofline needs the dominant kernel's own
// duration measured live on the launching stream).  Null = no events.
struct Profiler {
    virtual void begin(int kernel_id, cudaStream_t st) = 0;
    virtual void end(int kernel_id, cudaStream_t st) = 0;
    virtual ~Profiler() {}
};

// ---- launchers (gg_kernels.cu); every function enqueues on `st` and returns the number of
// kernel launches it issued (for gg_kernel_launches()). -----------------------------------
int launch_init_map(const View& v, int slot, float z, cudaStream_t st);
int launch_build_detect_table(const View& v, const CfgConst& c, float4* tab, cudaStream_t st);
int launch_roll(const View& v, const SlotParams* batch, int count, cudaStream_t st, Profiler* prof);
// layer_map: TMA descriptor of the handle's layer arena as a 3-D tensor (i, j, slot * n_layers + layer), box
// 40 x 12 x 1 (k_detect_tma); null -> the patch detection stages its tile with plain loads (N % 4 != 0)
int launch_scan_pipeline(const View& v, const SlotParams* batch, int count, int max_points, int stop_after, cudaStream_t st,
                         Profiler* prof, const CUtensorMap* layer_map);
// single phases / single cells (the reference's public per-phase methods)
// count_layer: the plane detection reads as "points"; recompute: the variance is L_M2 / (points + FLT_MIN) (:323),
// computed inside the detection kernel and stored to L_VARIANCE (full layers only)
int launch_detect_only(const View& v, const SlotParams* batch, int count, cudaStream_t st, Profiler* prof, const CUtensorMap* layer_map,
                       int count_layer, bool recompute);
int launch_spiral_only(const View& v, const SlotParams* batch, int count, cudaStream_t st, Profiler* prof);
int launch_interpolate_cell(const View& v, const CfgConst& c, int slot, int x, int y, cudaStream_t st);
int launch_detect_cell(const View& v, const CfgConst& c, int slot, int S, int i, int j, int count_layer, cudaStream_t st);
// The output cloud of `count` completed scans, compacted into dests[k] (dests[k] goes with batch[k]).
// compact: count + scan passes (needed for index / cloud / count); write: the write pass (needed for index / cloud /
// labels).  A batch that wants only labels needs only the write pass.
int launch_output(const View& v, const SlotParams* batch, const OutDest* dests, int count, int max_points, bool compact, bool write,
                  cudaStream_t st, Profiler* prof);
// Layers named in one gg_get_layers_to_device / gg_set_layers_from_device call, resolved once and passed by value.
// LAYER_POINTS stands for "points", whose layer depends on the slot (it travels with each scan, see launch_layer_copy).
constexpr int LAYER_POINTS = -1;
struct LayerList {
    int idx[L_NUM];  // [n] layer index (Layer) or LAYER_POINTS
    int n;
};
// Copies `count` slots' layers between the arena and the caller's buffer buf[k][l][N2] (plane l of scan k at
// (k * names.n + l) * N2), exporting (import = false: arena -> buf) or importing (import = true: buf -> arena).  Per
// scan the staging entry carries batch[s].slot, batch[s].pos = its position k in the call and batch[s].points_layer;
// every other field is zero.  buf must not overlap the arena.
int launch_layer_copy(const View& v, const SlotParams* batch, int count, const LayerList& names, float* buf, bool import, cudaStream_t st,
                      Profiler* prof);
// "next" rows of SURVEY.md section 8(f)
// f1: one PointCloud2 payload of a batch (gg_upload_cloud_msg[s], gg_run_cloud_msgs_to_device,
// gg_run_merged_cloud_msgs_to_device).  It sits in the staging entry next to the scans' SlotParams, in a parallel array
// with the same index (like OutDest).
struct UnpackDesc {
    const unsigned char* raw;  // msg.data on the device (the handle's staging copy or the caller's buffer)
    int point_step;
    int off[5];                // byte offsets of x, y, z, intensity, ring (-1: field absent)
    int transform;             // 0: frame_id == "map", copy only
    int first;                 // record of the slot's buffer where the payload's first point lands (one part of a merged scan)
    double T[12];              // row-major 3x4 [R|t] of lookupTransform("map", frame_id)
};
// PointCloud2 payloads -> PointXYZIR records in the map frame, for `count` payloads: descs[k] (batch[k].n_points records)
// lands in the slot's own cloud buffer at v.points + batch[k].slot * pcap + descs[k].first.
int launch_unpack(const View& v, const SlotParams* batch, const UnpackDesc* descs, int count, int max_points, cudaStream_t st, Profiler* prof);
// f3: the images of publish_grid_map_layer for `count` scans, with the staging entry of launch_layer_copy (batch[s].slot,
// batch[s].pos = position k in the call, batch[s].points_layer).
// launch_layer_images: plane l of scan k -> dst[(k * names.n + l) * N2] as N * N bytes, row-major (i, j); range (may be
// null) [k][l][2] = lower, upper.  partial: [n_slots][L_NUM][cdiv(N2, IMG_RANGE_CELLS)] scratch of the per-block
// ranges, indexed by slot (two calls that share a slot are ordered on the slot's stream).
constexpr int IMG_RANGE_CELLS = 4096;
int launch_layer_images(const View& v, const SlotParams* batch, int count, const LayerList& names, int2* partial, unsigned char* dst, float* range,
                        cudaStream_t st, Profiler* prof);
// launch_terrain_images: the terrain image of scan k -> dst[k][N][N][3] (needs the full layers)
int launch_terrain_images(const View& v, const SlotParams* batch, int count, float* dst, cudaStream_t st, Profiler* prof);
// f4: the evaluation tallies of the last completed scan of `count` slots, added into counts[k][EVAL_LABELS][2] (k =
// batch[s].pos, the scan's position in the call).  batch[s].n_points / src / packed describe the scan's input;
// max_points: the largest n_points of the batch.
int launch_eval(const View& v, const SlotParams* batch, int count, int max_points, unsigned long long* counts, cudaStream_t st, Profiler* prof);
constexpr int EVAL_LABELS = GG_EVAL_IDS;  // ring values (SemanticKITTI label ids <= 259) x {ground, non-ground}
// Terrain lookups (gg_sample_layers_to_device): one set of query positions of a slot and where its results go.  It sits
// in the staging entry next to the scans' SlotParams, in a parallel array with the same index (like OutDest).
struct QueryDesc {
    const unsigned char* data;  // batch[k].n_points records of point_step bytes, float32 x / y at off_x / off_y (map frame)
    float* dst;                 // [names.n][n]: value of name l at query q at dst[l * n + q]
    int32_t* cell;              // [n] i + j * N of the query's cell, -1 outside; null: none
    int point_step, off_x, off_y;
    int reserved;               // zero
};
// The values of `names` at the positions of descs[k] in the map of batch[k].slot at (batch[k].px, batch[k].py);
// mode GG_SAMPLE_NEAREST / GG_SAMPLE_LINEAR.  Per scan the staging entry carries slot, px, py, n_points (the set's size)
// and points_layer.  max_points: the largest n_points of the batch.
int launch_sample(const View& v, const SlotParams* batch, const QueryDesc* descs, int count, int max_points, const LayerList& names, int mode,
                  cudaStream_t st, Profiler* prof);
// Point classes and heights (gg_point_info_to_device): where one slot's results go.  It sits in the staging entry next
// to the slots' SlotParams, in a parallel array with the same index (like OutDest).
struct PointInfoDest {
    uint32_t* codes;   // [n] class << 24 | cell; null: none
    float* height;     // [n] z - ground[cell], NaN for absent points; null: none
};
// The codes and heights of the last scan of batch[k].slot into dests[k]; batch[k].n_points is that scan's point count
// (0: nothing to write).  max_points: the largest n_points of the batch.
int launch_point_info(const View& v, const SlotParams* batch, const PointInfoDest* dests, int count, int max_points, cudaStream_t st,
                      Profiler* prof);

// ---- poses from device memory (gg_update_poses_from_device) ----
// fp64 arithmetic, correctly rounded and never contracted, on the host and on the device
__host__ __device__ __forceinline__ double pose_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double pose_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ __forceinline__ double pose_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double pose_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// ---- the constants of one configuration (GroundSegmentation::setConfig, GroundGrid::setConfig) ----
// One derivation for the host (gg_set_slot_config, gg_set_config) and the device (k_store_configs), with the same
// correctly rounded fp64 operations, so both produce the same 120 bytes for the same gg_config.
__host__ __device__ __forceinline__ void derive_config(const gg_config& c, CfgConst& k) {
    k.max_ring = c.max_ring;
    k.pc_var_thresh_f = (float)c.point_count_cell_variance_threshold;
    k.min_outlier_conf = c.min_outlier_detection_ground_confidence;
    k.outlier_tol = c.outlier_tolerance;
    k.gp_thresh = c.ground_patch_detection_minimum_point_count_threshold;
    k.df_sq = pose_mul(c.distance_factor, c.distance_factor);
    k.mdf_sq = pose_mul(c.minimum_distance_factor, c.minimum_distance_factor);
    const double m10 = pose_mul(c.minimum_distance_factor, 10.0);
    k.mdf10_sq = pose_mul(m10, m10);
    k.psc_sq = pose_mul(c.patch_size_change_distance, c.patch_size_change_distance);
    k.occ_factor = c.occupied_cells_point_count_factor;
    k.occ_factor2 = pose_mul(c.occupied_cells_point_count_factor, (double)2.0f);
    k.dec_factor = c.occupied_cells_decrease_factor;
    k.lab_fac = pose_mul(c.minimum_distance_factor, 5.0);
    k.lab_thres = c.miminum_point_height_threshold;
    k.lab_obs = c.minimum_point_height_obstacle_threshold;
    // decay_confidence: o - o / dec_factor, floored at 0.001.  For factors >= 1 the exact value o * (1 - 1/F) grows
    // with o, so if the floor value 0.001f itself decays to clearly below 0.001, every confidence <= 0.001f ends on the
    // floor as well (rounding errors are ~1e-19, the margin asked for is 1e-6).
    const double o = (double)0.001f;
    const double dec = pose_sub(o, pose_div(o, k.dec_factor));
    k.decay_floor_ok = (k.dec_factor >= 1.0 && dec < 0.000999) ? 1 : 0;
    k.reserved = 0;
}

// ---- confidence decay of the spiral sweep (interpolate_cell :463-464), shared by every spiral path ----
// std::max(c - c / decrease_factor, 0.001) in fp64.  The result is >= 0.001 or NaN: +-inf decays to NaN (inf - inf),
// and so does NaN (std::max keeps its first argument when the comparison fails).
__host__ __device__ __forceinline__ float decay_confidence(const CfgConst& kc, float occ) {
    // Confidences sit at the 0.001 floor in most of the map; from there down to -FLT_MAX the result is the floor again
    // (host-checked for the configured factor, CfgConst::decay_floor_ok), which skips the fp64 division.  -inf is not
    // in that range: it decays to NaN like every other non-finite confidence.
    if (kc.decay_floor_ok && occ <= 0.001f && occ >= -FLT_MAX) return 0.001f;
    const double o = (double)occ;
    const double dec = pose_sub(o, pose_div(o, kc.dec_factor));
    return (float)((dec < 0.001) ? 0.001 : dec);
}
// The skewed spiral stores, per visit, the confidence the visit leaves (SD, written by k_detect): the decay of a cell
// beyond minDistSquared, SKEW_NEAR (never a decay) for a cell the visit does not decay.
constexpr float SKEW_NEAR = -1.0f;
__host__ __device__ __forceinline__ bool skew_decays(float d) { return d != SKEW_NEAR; }

// gg_host.cpp:move_map for one position, for a roll resolved on the device: the whole-cell shift toward (nx, ny),
// rounded half away from zero, and the map position advanced by it.  Returns 1 (the cells shift), 0 (no shift) or -1:
// a non-finite quotient or a shift outside int32 (move_map's int conversion is undefined there), which leaves px, py
// and the shift untouched.
__host__ __device__ __forceinline__ int resolve_move(double res, double& px, double& py, double nx, double ny, int& shift_i, int& shift_j) {
    const double tx = pose_div(pose_sub(nx, px), res), ty = pose_div(pose_sub(ny, py), res);
    const double rx = pose_add(tx, tx > 0 ? 0.5 : -0.5), ry = pose_add(ty, ty > 0 ? 0.5 : -0.5);
    // truncation toward zero lands in (-2^31, 2^31) and -cx fits as well; NaN fails every comparison
    if (!(rx > -2147483648.0 && rx < 2147483648.0 && ry > -2147483648.0 && ry < 2147483648.0)) return -1;
    const int cx = (int)rx, cy = (int)ry;
    shift_i = -cx;
    shift_j = -cy;
    px = pose_add(px, pose_mul((double)cx, res));
    py = pose_add(py, pose_mul((double)cy, res));
    return (cx != 0 || cy != 0) ? 1 : 0;
}

// ---- the outlier ray-march of k_rasterize past its first steps (insert_cloud :255-272) ----
// fp32 arithmetic, correctly rounded and never contracted, on the host and on the device
__host__ __device__ __forceinline__ float ray_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float ray_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// One point's ray after the pre-test (:244-257): the unit direction v (vz < -0.01f), len^2 and the map it walks.
struct OutlierRay {
    double px, py, half, res;  // map position, len / 2, resolution
    double len2;               // std::pow(len, 2.0)
    double thr, tol;           // min_outlier_detection_ground_confidence, outlier_tolerance
    float ox, oy, oz;          // cloud origin
    float vx, vy, vz;
    int N;
};

// What one step of the march computes from `step` (:258-262).  Each quantity is a monotone function of step:
// (float)step, fl(fs * v), fl(s + o), the index -trunc((p - len/2 - pos) / res), lhs and the height bound all are.
__host__ __device__ __forceinline__ int ray_trunc(double v) {
    // grid_map's cast<int>() of the quotient, clamped as k_rasterize's trunc_index clamps it (beyond +-1e9 the index is
    // outside the map either way; the clamp keeps it monotone)
    if (!(v == v)) return 1000000000;
    if (v > 1.0e9) return 1000000000;
    if (v < -1.0e9) return -1000000000;
    return (int)v;
}
// the cell index along axis a (0: x, 1: y) of step `step`
__host__ __device__ __forceinline__ int ray_index(const volatile OutlierRay& r, unsigned step, int a) {
    const float s = ray_mul((float)step, a ? r.vy : r.vx);
    const double p = (double)ray_add(s, a ? r.oy : r.ox);
    return -ray_trunc(pose_div(pose_sub(pose_sub(p, r.half), a ? r.py : r.px), r.res));
}
// lhs < len2: the loop still runs at `step`
__host__ __device__ __forceinline__ bool ray_runs(const volatile OutlierRay& r, unsigned step) {
    const float fs = (float)step;
    const float sx = ray_mul(fs, r.vx), sy = ray_mul(fs, r.vy), sz = ray_mul(fs, r.vz);
    return pose_add(pose_add(pose_mul((double)sx, (double)sx), pose_mul((double)sy, (double)sy)), pose_mul((double)sz, (double)sz)) < r.len2;
}

// The first step t in [lo, hi) with d0 * ix(t) > b0 or d1 * iy(t) > b1, hi if there is none (d = 0: that axis is not
// tested).  d0 * ix and d1 * iy do not decrease along the ray, so the predicate is false up to some step and true from
// there on.
__host__ __device__ __forceinline__ unsigned ray_first(const volatile OutlierRay& r, unsigned lo, unsigned hi, int d0, int b0, int d1, int b1) {
    while (lo < hi) {
        const unsigned mid = lo + (hi - lo) / 2;
        if ((d0 && d0 * ray_index(r, mid, 0) > b0) || (d1 && d1 * ray_index(r, mid, 1) > b1))
            hi = mid;
        else
            lo = mid + 1;
    }
    return lo;
}

// The march from step `from` on, without walking it step by step: true when some step in [from, S) finds an occluding
// cell, S being the first step whose lhs reaches len2.  The cells the ray visits are a monotone staircase and the steps
// of one cell form an interval; the cell tests (interior, the clamped 3x3 sum, C > 0.01f) do not depend on the step and
// the height bound fl(fl(fs * vz) + oz) + tol does not increase along the ray, so a cell occludes at some step of its
// interval exactly when it does at the interval's last step.  The walk finds S, the interior part of the ray and each
// cell's last step by bisection over step: O(cells * 31) instead of O(steps).
// The reference counts in `int step`; a ray whose loop would run past INT_MAX overflows it (undefined behaviour).  Here
// the march ends after step INT_MAX, as if the loop condition failed there.
// G / C: the prior's "ground" / "groundpatch" (column-major, N x N, N > 4).  k_rasterize keeps r in local memory (it is
// volatile here) and runs the walk inline, so that the walk's few registers fit beside the kernel's.
__host__ __device__ __forceinline__ bool outlier_walk(const volatile OutlierRay& r, const float* G, const float* C, unsigned from) {
    const unsigned end = 2147483648u;  // one past INT_MAX
    if (from >= end) return false;
    unsigned lo = from, hi = end;
    while (lo < hi) {  // S: lhs does not decrease along the ray
        const unsigned mid = lo + (hi - lo) / 2;
        if (ray_runs(r, mid))
            lo = mid + 1;
        else
            hi = mid;
    }
    const unsigned S = lo;
    if (S <= from) return false;
    const int N = r.N;
    const int d0 = ray_index(r, S - 1, 0) >= ray_index(r, from, 0) ? 1 : -1;
    const int d1 = ray_index(r, S - 1, 1) >= ray_index(r, from, 1) ? 1 : -1;
    // interior steps (0 < ix < N-1 and 0 < iy < N-1): an interval per axis, so an interval
    unsigned s = ray_first(r, from, S, d0, d0 > 0 ? 0 : 1 - N, 0, 0);
    const unsigned s1 = ray_first(r, from, S, 0, 0, d1, d1 > 0 ? 0 : 1 - N);
    s = s > s1 ? s : s1;
    unsigned e = ray_first(r, from, S, d0, d0 > 0 ? N - 2 : -1, 0, 0);
    const unsigned e1 = ray_first(r, from, S, 0, 0, d1, d1 > 0 ? N - 2 : -1);
    e = e < e1 ? e : e1;
    while (s < e) {
        const int ix = ray_index(r, s, 0), iy = ray_index(r, s, 1);
        s = ray_first(r, s + 1, e, d0, d0 * ix, d1, d1 * iy);  // one past the cell's last step
        const int r0 = ix - 1 > 2 ? ix - 1 : 2, c0 = iy - 1 > 2 ? iy - 1 : 2;  // :268 (clamped, not centred)
        const float* B = C + r0 + (size_t)c0 * N;
        const size_t n = N;
        // Eigen 3.3.7's binary split over the column-major block (k_rasterize's tree9)
        const float bs = ray_add(ray_add(ray_add(B[0], B[1]), ray_add(B[2], B[n])),
                                 ray_add(ray_add(B[n + 1], B[n + 2]), ray_add(B[2 * n], ray_add(B[2 * n + 1], B[2 * n + 2]))));
        const size_t cell = (size_t)ix + (size_t)iy * n;
        // the height bound at the cell's last step, the lowest of the cell
        if ((double)bs > r.thr && C[cell] > 0.01f && (double)G[cell] >= pose_add((double)ray_add(ray_mul((float)(s - 1), r.vz), r.oz), r.tol))
            return true;
    }
    return false;
}
// The plain loop hands a ray to outlier_walk at this step (physical rays end long before it).
constexpr int RAY_WALK_FROM = 4096;

// Per-record bits of a staging entry (PoseBits[m] next to its SlotParams): where k_stage_poses takes the record's
// pose from.
enum PoseBits : int {
    POSE_POSITION = 1,   // px / py from the slot's entry of the device position table (the position is device-owned)
    POSE_ORIGIN = 2,     // ox / oy / oz / base_z_f from the slot's device scan pose (GG_SCAN_DEVICE_POSE)
    POSE_COUNT = 4,      // a scan of GG_SCAN_DEVICE_COUNT: n_points (staged: the capacity) from the slot's stored count,
                         // 0 when that is outside [0, capacity); the result also goes to the slot's last count
    POSE_LAST_COUNT = 8, // n_points from the slot's last count (the count of its last scan is device-owned)
    POSE_PART_COUNTS = 16,  // a merged scan of GG_SCAN_DEVICE_PART_COUNTS: k_stage_parts (not k_stage_poses) resolves
                            // its parts' counts and offsets from the slot's stored part counts
    POSE_CONFIG = 32,    // cfg from the slot's entry of ConfigTables::cfg (the slot is device-configured; its detect_tab
                         // is staged from the host: the slot's private table)
    POSE_MASK = 64,      // a scan of GG_SCAN_DEVICE_MASK: skip = (the slot's stored mask == 0); a skipped scan runs on 0 points,
                         // and the slot's last count becomes the scan's resolved count (0 when skipped)
};
// The handle's per-slot configurations from device memory (allocated on the first gg_set_slot_configs_from_device).
struct ConfigTables {
    gg_config* raw;      // [n_slots] the configuration as the caller gave it (gg_get_slot_config returns it)
    CfgConst* cfg;       // [n_slots] its derived constants
};
// The handle's per-slot device tables (allocated on the first gg_update_poses_from_device).
struct PoseTables {
    double2* position;   // [n_slots] map position of a device-owned slot
    float4* scan_pose;   // [n_slots] origin x, y, z and (float)base_z
};
// The handle's per-slot point counts from device memory (allocated on the first gg_set_point_counts_from_device).
struct CountTables {
    int32_t* stored;     // [n_slots] the latest count gg_set_point_counts_from_device stored, as the caller gave it
    int32_t* last;       // [n_slots] the count the slot's last GG_SCAN_DEVICE_COUNT scan ran on
    int32_t* parts;      // [n_slots][GG_MAX_CLOUD_PARTS] the latest part counts gg_set_part_counts_from_device stored
                         // (allocated on its first call)
    int32_t* mask;       // [n_slots] the latest scan mask gg_set_scan_masks_from_device stored, as the caller gave it
                         // (allocated on its first call)
};
// Patches the `count` records of batch whose bits ask for it from the tables; runs after the entry's copy and before
// the kernels that read it.
int launch_stage_poses(const PoseTables& t, const CountTables& c, const CfgConst* cfgs, SlotParams* batch, const int* bits, int count,
                       cudaStream_t st, Profiler* prof);
// Configurations from device memory (gg_set_slot_configs_from_device), two launches on one staging entry whose record j
// carries slot, pos and detect_tab (the slot's private table).  k_store_configs, one thread per record: unless mask (may
// be null) is zero at pos, cfg[pos] goes to the slot's entry of t.raw and its derivation (derive_config) to t.cfg; the
// record's n_points becomes 1 if it was reconfigured, else 0.  k_rebuild_detect_tables, a grid of (cells, records):
// each reconfigured record's detect table is rebuilt from t.cfg; the blocks of the other records exit after one load.
int launch_store_configs(const View& v, const ConfigTables& t, SlotParams* batch, int count, const gg_config* cfg, const int32_t* mask,
                         cudaStream_t st, Profiler* prof);
// One thread per record: the count of batch[j] (at dev_n[batch[j].pos]) into the slot's entry of `table` (c.stored for
// gg_set_point_counts_from_device, c.mask for gg_set_scan_masks_from_device).
int launch_store_counts(int32_t* table, const SlotParams* batch, int count, const int32_t* dev_n, cudaStream_t st, Profiler* prof);
// One thread per record: the parts_per_slot part counts of batch[j] (at dev_n[batch[j].pos * parts_per_slot]) into the
// slot's row of c.parts.
int launch_store_part_counts(const CountTables& c, const SlotParams* batch, int count, const int32_t* dev_n, int parts_per_slot, cudaStream_t st,
                             Profiler* prof);
// The part rounds of one scan entry of gg_run_merged_cloud_msgs_to_device: record j of round p's entry is part p of the
// entry's scan j (n_points = the part's capacity, 0 without one; descs[j].first = the capacities before it).  Null: the
// round has no part to read and is not launched.
struct PartRounds {
    SlotParams* params[GG_MAX_CLOUD_PARTS];
    UnpackDesc* descs[GG_MAX_CLOUD_PARTS];
};
// One thread per record of the scan entry whose bits hold POSE_PART_COUNTS: per part p the count u_p = v_p if
// 0 <= v_p <= capacity, else 0 (v_p: the slot's stored part count), written into round p's record with the offset
// u_0 + ... + u_{p-1}; the scan record's n_points and the slot's last count become the sum.  A record that k_stage_poses
// skipped (POSE_MASK) gets u_p = 0 for every part, so no part of it is unpacked.  Runs after k_stage_poses and the
// entries' copies, and before the rounds.
int launch_stage_parts(const CountTables& c, SlotParams* batch, const int* bits, int count, const PartRounds& rounds, cudaStream_t st,
                       Profiler* prof);
// The poses of one gg_update_poses_from_device call (entry batch[j].pos of each array); null xy: no roll, null origin:
// no scan pose.
struct DevicePoses {
    const double* xy;
    const double* T;
    const float* origin;
    const double* base_z;
    int32_t* moved;
};
// One thread per record: resolves the roll of batch[j] from its staged position (bits POSE_POSITION: the device table's),
// writes shift_i / shift_j, px / py and t20..t23 into the record for launch_roll, the new position into the table and
// moved[pos]; stores the scan pose.
int launch_pose_resolve(const View& v, const PoseTables& t, SlotParams* batch, const int* bits, int count, const DevicePoses& in, cudaStream_t st,
                        Profiler* prof);
// Map resets (gg_init_maps_from_device): record j re-initialises the layers of batch[j].slot as k_init_map does at the
// odometry xyz[batch[j].pos] and writes its x, y into the position table, unless mask (may be null) is zero at pos; a
// masked-off record whose bits lack POSE_POSITION seeds its staged px / py into the table instead.
int launch_reset_maps(const View& v, const PoseTables& t, const SlotParams* batch, const int* bits, int count, const double* xyz, const int32_t* mask,
                      cudaStream_t st, Profiler* prof);
// Map snapshots (gg_save_maps_to_device, gg_restore_maps_from_device): records of snapshot_bytes(N2p) bytes, the
// gg_map_snapshot header followed by "ground" at byte 64 and "groundpatch" at 64 + 4 * n2p.
constexpr int SNAPSHOT_HEADER = 64;
static_assert(sizeof(gg_map_snapshot) == SNAPSHOT_HEADER, "gg_map_snapshot is the 64-byte header of a snapshot");
__host__ __device__ constexpr int snapshot_cells(int N2) { return (N2 + 3) & ~3; }
__host__ __device__ constexpr size_t snapshot_bytes(int N2) { return SNAPSHOT_HEADER + (size_t)8 * snapshot_cells(N2); }
struct SnapshotPool {
    const unsigned char* records;  // [n_pool][snapshot_bytes]
    const int32_t* index;          // [count] or null (= pos)
    int32_t* status;               // [count] or null
    int n_pool;
    uint32_t res_bits;             // the handle's float resolution, bitwise
};
struct SnapshotDest {
    unsigned char* records;        // [count][snapshot_bytes]
    const int32_t* mask;           // [count] or null
    uint32_t res_bits;
};
// Restore: the snapshot-taking instantiation of k_reset_maps.  Record j takes "ground" and "groundpatch" from the pool
// record index[pos] (pos when index is null), every other layer starts as k_init_map starts it, and the record's position
// goes to the table; status[pos] = 1.  An index outside [0, n_pool) (status 0) or a record whose header does not match
// the handle (status -1) leaves the slot untouched, and a host-owned position (bits lack POSE_POSITION) is seeded from the
// staged px / py, as a masked-off reset seeds it.
int launch_restore_maps(const View& v, const PoseTables& t, const SlotParams* batch, const int* bits, int count, const SnapshotPool& pool,
                        cudaStream_t st, Profiler* prof);
// Save (k_save_maps): record j writes the header (position from the table when bits hold POSE_POSITION, else the staged
// px / py) and both planes of its slot into records[pos], unless mask is zero at pos.
int launch_save_maps(const View& v, const PoseTables& t, const SlotParams* batch, const int* bits, int count, const SnapshotDest& dst,
                     cudaStream_t st, Profiler* prof);

// ---- step plans (gg_step_plan_create) ----
// One thread per record: descs[j] takes the 12 doubles at T[j] as its transform (transform = 1) when T[j] is given, and
// is left alone otherwise.  Runs on a replay's working records, before k_unpack_transform reads them.
int launch_stage_transforms(UnpackDesc* descs, const double* const* T, int count, cudaStream_t st);
// The dynamic shared-memory opt-in of the spiral kernel launch_scan_pipeline picks for v (it sets it at launch time
// too; a recorded step sets it before the recording).
int prepare_scan_pipeline(const View& v);

}  // namespace gg
