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
};

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

// Per-record bits of a staging entry (PoseBits[m] next to its SlotParams): where k_stage_poses takes the record's
// pose from.
enum PoseBits : int {
    POSE_POSITION = 1,   // px / py from the slot's entry of the device position table (the position is device-owned)
    POSE_ORIGIN = 2,     // ox / oy / oz / base_z_f from the slot's device scan pose (GG_SCAN_DEVICE_POSE)
};
// The handle's per-slot device tables (allocated on the first gg_update_poses_from_device).
struct PoseTables {
    double2* position;   // [n_slots] map position of a device-owned slot
    float4* scan_pose;   // [n_slots] origin x, y, z and (float)base_z
};
// Patches the `count` records of batch whose bits ask for it from the tables; runs after the entry's copy and before
// the kernels that read it.
int launch_stage_poses(const PoseTables& t, SlotParams* batch, const int* bits, int count, cudaStream_t st, Profiler* prof);
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

}  // namespace gg
