// groundgrid_b200 -- hand-written sm_90a (H100) kernels of the GroundGrid per-scan hot path.
//
// Phases (reference: src/GroundSegmentation.cpp, see DESIGN.md for the data layout):
//   k_rasterize     point -> cell, ignore test, outlier ray-march; every warp claims, per cell it
//                   touches, one contiguous run of the cell's segment (one atomic per run)     (:200-280)
//   k_cell_tiles/place  exclusive scan of the per-cell counts -> segment starts; worklist of non-empty cells by count class
//   k_scatter       z of every kept point -> its slot of the cell's segment, run descriptors
//   k_cell_stats    per-cell sequential count / min / Welford mean+M2 -> variance, walking the
//                   runs of a cell in input order (the Welford recurrence of :298-305 is order
//                   dependent)                                                                 (:282-309,323)
//   k_detect        3x3 / 5x5 ground-patch stencil updating G, C              (:314-395)
//   k_spiral        level-scheduled wavefront of the in-place spiral sweep    (:398-465)
//   k_label         per-point ground / non-ground decision                    (:146-196)
//   k_out_*         output cloud order: kept, ignored, outliers               (:112-117,150,185)
//   k_roll_*        GroundGrid::update: whole-cell roll + seeding             (GroundGrid.cpp:83-147)
//
// Arithmetic rules (SURVEY.md App. A): no FMA contraction (compiled with --fmad=false AND
// written with __f*_rn intrinsics where a product feeds a sum), IEEE division / sqrt,
// fp64 wherever the reference's C++ promotes to double, Eigen 3.3.7's binary-split
// reduction order for every fixed-size block sum.
#include <cuda.h>   // CUtensorMap (the descriptor is encoded on the host, gg_capi.cu)

#include <cfloat>
#include <cstddef>
#include <cstdio>

#include "gg_internal.h"

namespace gg {

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int trunc_index(double v) {
    // grid_map: indexVector.cast<int>() (truncation toward zero); clamped so that NaN / huge
    // values map far outside instead of being undefined.
    if (!(v == v)) return 1000000000;
    if (v > 1.0e9) return 1000000000;
    if (v < -1.0e9) return -1000000000;
    return __double2int_rz(v);
}

// trunc(a / res) exactly as the IEEE division would give it, without paying for the division in the
// common case: q = a * (1 / res) differs from the correctly rounded quotient by a few ulp
// (|q| < 1e6 here, so < 1e-9 absolute); whenever q is farther than 1e-6 from every integer, no
// integer lies between the two values and trunc(q) == trunc(a / res).  Otherwise (a point within
// a micro-cell of a cell boundary, or a huge / non-finite value) the real division decides.
__device__ __forceinline__ int trunc_quotient(double a, double res, double rres) {
    const double q = __dmul_rn(a, rres);
    const double f = __dsub_rn(q, rint(q));
    if (fabs(q) < 1.0e6 && fabs(f) > 1.0e-6) return __double2int_rz(q);
    return trunc_index(__ddiv_rn(a, res));
}

// grid_map_core getIndexFromPosition with start index (0,0): -(int)((p - len/2 - pos) / res)
__device__ __forceinline__ void grid_index(const Const& k, double px, double py, double x, double y, int& ix, int& iy) {
    ix = -trunc_quotient(__dsub_rn(__dsub_rn(x, k.half), px), k.res, k.rres);
    iy = -trunc_quotient(__dsub_rn(__dsub_rn(y, k.half), py), k.res, k.rres);
}

// grid_map_core checkIfPositionWithinMap: t = -(p - pos - len/2); 0 <= t < len
__device__ __forceinline__ bool grid_inside(const Const& k, double px, double py, double x, double y) {
    const double tx = -__dsub_rn(__dsub_rn(x, px), k.half);
    const double ty = -__dsub_rn(__dsub_rn(y, py), k.half);
    return tx >= 0.0 && ty >= 0.0 && tx < k.len && ty < k.len;
}

// grid_map getPositionFromIndex along one axis (start index (0,0)): pos + (len/2 - res/2) + res * (-(double)index)
__device__ __forceinline__ double cell_centre(const Const& k, double pos, int index) {
    const double off = __dsub_rn(k.half, __dmul_rn(0.5, k.res));
    return __dadd_rn(__dadd_rn(pos, off), __dmul_rn(k.res, (double)(-index)));
}

// Eigen 3.3.7 redux_novec_unroller: binary split over the block's coefficients (column-major).
template <int Start, int Len>
struct TreeSum {
    template <typename F>
    __device__ __forceinline__ static float run(const F& e) {
        return __fadd_rn(TreeSum<Start, Len / 2>::run(e), TreeSum<Start + Len / 2, Len - Len / 2>::run(e));
    }
};
template <int Start>
struct TreeSum<Start, 1> {
    template <typename F>
    __device__ __forceinline__ static float run(const F& e) {
        return e(Start);
    }
};

__device__ __forceinline__ float tree9(const float* e) {
    return __fadd_rn(__fadd_rn(__fadd_rn(e[0], e[1]), __fadd_rn(e[2], e[3])),
                     __fadd_rn(__fadd_rn(e[4], e[5]), __fadd_rn(e[6], __fadd_rn(e[7], e[8]))));
}

__device__ __forceinline__ int warp_inclusive_scan(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// Exclusive scan of n ints (in -> out, may alias) by one block of 1024 threads: tiles of 4096
// elements, 4 consecutive ints per thread (coalesced), next tile prefetched while the current
// one is scanned.  Returns the grand total to every thread.
template <int STRIDE = 1>
__device__ int block_exclusive_scan_1024(const int* in, int* out, int n) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    int nx[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) nx[q] = (tid * 4 + q < n) ? in[(size_t)(tid * 4 + q) * STRIDE] : 0;
    __syncthreads();
    for (int base = 0; base < n; base += 4096) {
        int cur[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) cur[q] = nx[q];
        const int nb = base + 4096 + tid * 4;
#pragma unroll
        for (int q = 0; q < 4; ++q) nx[q] = (nb + q < n) ? in[(size_t)(nb + q) * STRIDE] : 0;
        const int sum = cur[0] + cur[1] + cur[2] + cur[3];
        const int incl = warp_inclusive_scan(sum);
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const int w = s_warp[lane];
            const int wi = warp_inclusive_scan(w);
            s_warp[lane] = wi - w;
        }
        __syncthreads();
        const int carry = s_carry;
        int run = carry + s_warp[warp] + incl - sum;
        const int idx = base + tid * 4;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (idx + q < n) out[idx + q] = run;
            run += cur[q];
        }
        __syncthreads();
        if (tid == 1023) s_carry = run;
        __syncthreads();
    }
    return s_carry;
}

// ------------------------------------------------------------------------------------------
// fills / map init / roll
// ------------------------------------------------------------------------------------------
// GroundGrid::update (GroundGrid.cpp:96-133,143): new(r, c) = old(r + shift_i, c + shift_j);
// exposed cells: ground = -(T * (cx, cy, 0)).z in fp64, groundpatch = 0.
// Four consecutive cells per thread: the eight (shifted, hence unaligned but contiguous) loads are issued together and,
// when N*N is a multiple of 4 (every layer then starts 16-byte aligned), the results leave as 16-byte stores.
constexpr int ROLL_ILP = 4;

__global__ void __launch_bounds__(256) k_roll_gather(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.y];
    if (sp.shift_i == 0 && sp.shift_j == 0) return;
    const Const& k = v.k;
    const int cell0 = (blockIdx.x * 256 + threadIdx.x) * ROLL_ILP;
    if (cell0 >= k.N2) return;
    const int N = k.N;
    const float* G = v.layer(sp.slot, L_GROUND);
    const float* C = v.layer(sp.slot, L_GROUNDPATCH);
    float* sg = v.roll_scratch + (size_t)sp.slot * 2 * k.N2;
    float* sc = sg + k.N2;
    float g[ROLL_ILP], c[ROLL_ILP];
    bool seed[ROLL_ILP];
#pragma unroll
    for (int u = 0; u < ROLL_ILP; ++u) {
        const int cell = cell0 + u;
        const int r = cell % N, cc = cell / N;
        const int orr = r + sp.shift_i, occ = cc + sp.shift_j;
        const bool live = cell < k.N2;
        seed[u] = live && !(orr >= 0 && orr < N && occ >= 0 && occ < N);
        const bool ld = live && !seed[u];
        g[u] = ld ? G[orr + occ * N] : 0.0f;
        c[u] = ld ? C[orr + occ * N] : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < ROLL_ILP; ++u)
        if (seed[u]) {
            const int cell = cell0 + u;
            const int r = cell % N, cc = cell / N;
            const double x = cell_centre(k, sp.px, r);
            const double y = cell_centre(k, sp.py, cc);
            // tf2::Transform * Vector3(x, y, 0): row2.dot(v) + origin.z
            const double tz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sp.t20, x), __dmul_rn(sp.t21, y)), __dmul_rn(sp.t22, 0.0)), sp.t23);
            g[u] = (float)(-tz);
            c[u] = 0.0f;
        }
    if ((k.N2 & 3) == 0) {
        *reinterpret_cast<float4*>(sg + cell0) = make_float4(g[0], g[1], g[2], g[3]);
        *reinterpret_cast<float4*>(sc + cell0) = make_float4(c[0], c[1], c[2], c[3]);
    } else {
#pragma unroll
        for (int u = 0; u < ROLL_ILP; ++u)
            if (cell0 + u < k.N2) {
                sg[cell0 + u] = g[u];
                sc[cell0 + u] = c[u];
            }
    }
}

__global__ void __launch_bounds__(256) k_roll_commit(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.y];
    if (sp.shift_i == 0 && sp.shift_j == 0) return;
    const int N2 = v.k.N2;
    const int cell0 = (blockIdx.x * 256 + threadIdx.x) * ROLL_ILP;
    if (cell0 >= N2) return;
    const float* sg = v.roll_scratch + (size_t)sp.slot * 2 * N2;
    float* G = v.layer(sp.slot, L_GROUND);
    float* C = v.layer(sp.slot, L_GROUNDPATCH);
    if ((N2 & 3) == 0) {
        const float4 a = *reinterpret_cast<const float4*>(sg + cell0);
        const float4 b = *reinterpret_cast<const float4*>(sg + N2 + cell0);
        *reinterpret_cast<float4*>(G + cell0) = a;
        *reinterpret_cast<float4*>(C + cell0) = b;
    } else {
#pragma unroll
        for (int u = 0; u < ROLL_ILP; ++u)
            if (cell0 + u < N2) {
                G[cell0 + u] = sg[cell0 + u];
                C[cell0 + u] = sg[N2 + cell0 + u];
            }
    }
}

// ------------------------------------------------------------------------------------------
// phase 1a: per-point rasterisation front end (insert_cloud up to the accumulate step)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rasterize_point(const View& v, const SlotParams& sp, int i, float& zout) {
    const Const& k = v.k;
    const CfgConst& kc = sp.cfg;
    const int N = k.N;
    const size_t base = (size_t)sp.slot * v.pcap;

    float x, y, z;
    int ring;
    if (sp.packed) {
        // packed SoA cloud: four fully coalesced streams, 14 bytes per point
        const int n_pad = (sp.n_points + 7) & ~7;
        x = __ldg(sp.packed + i);
        y = __ldg(sp.packed + n_pad + i);
        z = __ldg(sp.packed + 2 * n_pad + i);
        ring = (int)__ldg(reinterpret_cast<const unsigned short*>(sp.packed + 3 * n_pad) + i);
    } else {
        // coalesced 2 x 16-byte loads of the 32-byte PointXYZIR record
        const uint4* rec = reinterpret_cast<const uint4*>(sp.src + i);
        const uint4 a = __ldg(rec);
        const uint4 b = __ldg(rec + 1);
        x = __uint_as_float(a.x), y = __uint_as_float(a.y), z = __uint_as_float(a.z);
        ring = (int)(b.y & 0xffffu);
    }
    const float ox = sp.ox, oy = sp.oy, oz = sp.oz;

    const float dxo = __fsub_rn(x, ox), dyo = __fsub_rn(y, oy);
    // std::pow(dx, 2.0) + std::pow(dy, 2.0) in double (:223); the same sum feeds hypotf (:170)
    const double sq = __dadd_rn(__dmul_rn((double)dxo, (double)dxo), __dmul_rn((double)dyo, (double)dyo));
    const float sqdist = (float)sq;
    v.dist[base + i] = (float)__dsqrt_rn(sq);  // glibc hypotf: (float) sqrt((double)x*x + (double)y*y)

    uint32_t key = (uint32_t)k.N2;  // sentinel: not rasterised
    uint32_t code = PC_ABSENT << 24;

    const double px = sp.px, py = sp.py;
    int g0, g1;
    grid_index(k, px, py, (double)x, (double)y, g0, g1);
    if (grid_inside(k, px, py, (double)x, (double)y) && g0 >= 0 && g1 >= 0 && g0 < N && g1 < N) {
        const int cell = g0 + g1 * N;
        const bool border = (N <= g0 + 3) || (N <= g1 + 3);  // :167
        if (k.full_layers) atomicAdd(v.raw_i + (size_t)sp.slot * k.N2 + cell, 1);  // pointsRaw, :234
        if (ring > kc.max_ring || sqdist < 12.0f) {  // :237
            code = ((border ? PC_IGNORED_BORDER : PC_IGNORED) << 24) | (uint32_t)cell;
        } else {
            const float* G = v.layer(sp.slot, L_GROUND);
            const float* C = v.layer(sp.slot, L_GROUNDPATCH);
            bool outlier = false;
            const float oldg = G[cell];
            if ((double)z < __dsub_rn((double)oldg, 0.2)) {  // :244
                float vx = dxo, vy = dyo, vz = __fsub_rn(z, oz);
                const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz)));
                vx = __fdiv_rn(vx, len);
                vy = __fdiv_rn(vy, len);
                vz = __fdiv_rn(vz, len);
                const double len2 = __dmul_rn((double)len, (double)len);
                if (vz < -0.01f) {
                    // len is finite here (a non-finite one makes vz NaN or -0), so the loop ends; a ray still running
                    // at RAY_WALK_FROM is finished by the exact walk, whatever its length
                    bool walk = false;
                    for (int step = 3;; ++step) {
                        if (step == RAY_WALK_FROM) {
                            walk = true;
                            break;
                        }
                        const float fs = (float)step;
                        const float sx = __fmul_rn(fs, vx), sy = __fmul_rn(fs, vy), sz = __fmul_rn(fs, vz);
                        const double lhs = __dadd_rn(__dadd_rn(__dmul_rn((double)sx, (double)sx), __dmul_rn((double)sy, (double)sy)),
                                                     __dmul_rn((double)sz, (double)sz));
                        if (!(lhs < len2)) break;
                        int ix, iy;
                        grid_index(k, px, py, (double)__fadd_rn(sx, ox), (double)__fadd_rn(sy, oy), ix, iy);
                        if (ix <= 0 || iy <= 0 || ix >= N - 1 || iy >= N - 1) continue;
                        const int r0 = max(ix - 1, 2), c0 = max(iy - 1, 2);  // :268 (clamped, not centred)
                        float e[9];
#pragma unroll
                        for (int q = 0; q < 9; ++q) e[q] = C[(r0 + q % 3) + (c0 + q / 3) * N];
                        const float bs = tree9(e);
                        if ((double)bs > kc.min_outlier_conf && C[ix + iy * N] > 0.01f &&
                            (double)G[ix + iy * N] >= __dadd_rn((double)__fadd_rn(sz, oz), kc.outlier_tol)) {
                            outlier = true;
                            break;
                        }
                    }
                    if (walk) {
                        // the ray's constants stay in local memory while the walk runs (see outlier_walk)
                        volatile OutlierRay ray;
                        ray.px = px, ray.py = py, ray.half = k.half, ray.res = k.res, ray.len2 = len2;
                        ray.thr = kc.min_outlier_conf, ray.tol = kc.outlier_tol;
                        ray.ox = ox, ray.oy = oy, ray.oz = oz, ray.vx = vx, ray.vy = vy, ray.vz = vz, ray.N = N;
                        outlier = outlier_walk(ray, G, C, RAY_WALK_FROM);
                    }
                }
            }
            if (outlier) {
                code = (PC_OUTLIER << 24) | (uint32_t)cell;
            } else {
                key = (uint32_t)cell;
                code = ((border ? PC_KEPT_BORDER : PC_KEPT) << 24) | (uint32_t)cell;
            }
        }
    }
    v.code[base + i] = code;
    zout = z;
    return key;
}

// Words that travel from k_rasterize to k_scatter:
//   zw[i]   = (z bits, position inside the cell's segment | run-head flag in bit 31)      every point
//   runj[i] = arrival number of the run among the cell's runs | (run length - 1) << 26     run heads only
constexpr uint32_t RUN_LOW26 = (1u << 26) - 1u;

// RASTER_TILE consecutive points per block, RASTER_THREADS threads, thread order == point order inside a round, so
// the 32 lanes of a warp always hold 32 CONSECUTIVE points (point index >> 5 is warp-uniform: the "run id").
// Kept points of a warp that fall into the same cell form one run: the lowest lane claims `len` consecutive
// positions of the cell's segment and the run's directory entry with ONE 64-bit atomicAdd (low word: points of the
// cell, high word: runs of the cell); lane order inside the run is input order.  Runs of one cell never interleave
// (different warps own disjoint index ranges), so input order inside a cell = runs sorted by run id -- which
// k_cell_stats restores from the (few) directory entries without any sort pass over the points.
__global__ void __launch_bounds__(RASTER_THREADS, 5) k_rasterize(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.y];
    const int n = sp.n_points;
    const int tile0 = blockIdx.x * RASTER_TILE;
    if (tile0 >= n) return;
    const size_t base = (size_t)sp.slot * v.pcap;
    unsigned long long* cnt = v.cnt64 + (size_t)sp.slot * v.k.N2;
    const int lane = threadIdx.x & 31;
    const uint32_t lt_mask = (1u << lane) - 1u;
    for (int r = 0; r < RASTER_TILE / RASTER_THREADS; ++r) {
        const int i = tile0 + r * RASTER_THREADS + threadIdx.x;
        if (__all_sync(0xffffffffu, i >= n)) break;
        uint32_t key = (uint32_t)v.k.N2;
        float z = 0.0f;
        if (i < n) key = rasterize_point(v, sp, i, z);
        const bool kept = key != (uint32_t)v.k.N2;
        // lanes without a kept point get a private pseudo key (never equal to a cell id)
        const uint32_t peers = __match_any_sync(0xffffffffu, kept ? key : (0x80000000u | (uint32_t)lane));
        const int leader = __ffs(peers) - 1;
        const int len = __popc(peers);
        const bool head = kept && lane == leader;
        unsigned long long old = 0ull;
        if (head) old = atomicAdd(cnt + key, (1ull << 32) | (unsigned long long)len);
        const int start = __shfl_sync(0xffffffffu, (int)(uint32_t)old, leader);
        if (i < n) {
            const uint32_t w = kept ? ((uint32_t)(start + __popc(peers & lt_mask)) | (head ? 0x80000000u : 0u)) : 0u;
            v.zw[base + i] = make_uint2(__float_as_uint(z), w);
            if (head) v.runj[base + i] = ((uint32_t)(old >> 32) & RUN_LOW26) | ((uint32_t)(len - 1) << 26);
        }
    }
}

// ------------------------------------------------------------------------------------------
// phase 1b: segment starts (exclusive scan of the per-cell point counts), then every kept z goes to its
// position and every run head files the run in the cell's directory
// ------------------------------------------------------------------------------------------
// Count classes of the cell worklist: exact up to 32 points, then steps of 1/4 octave (cells of one class differ by
// less than 20 % in their walk length); heaviest class first.
constexpr int WL_CLASSES = 64;
__device__ __forceinline__ int worklist_class(int c) {
    if (c <= 32) return c;                                  // 1 .. 32 exact (0 never enters the list)
    const int e = 31 - __clz(c);                            // floor(log2 c) >= 5
    const int q = (c >> (e - 2)) & 3;                       // two bits below the leading one
    const int k = 33 + (e - 5) * 4 + q;
    return k < WL_CLASSES ? k : WL_CLASSES - 1;
}

// Segment starts and worklist in two short, fully parallel launches over tiles of CELL_TILE cells (a single block
// per scan would be a long serial chain):
//   k_cell_tiles   per tile: kept points and cells per count class            -> cell_agg[scan][tile][0 .. WL_CLASSES]
//   k_cell_place   per tile: prefix over the earlier tiles' aggregates, local exclusive scan -> cellstart; every
//                  non-empty cell goes to the scan's worklist, grouped by class (heaviest class first) so that the 32
//                  cells a warp of k_cell_stats walks have (almost) the same length.  The order inside a class is
//                  arbitrary -- every cell's result is independent of it.
constexpr int CELL_TILE = 4096;      // CT_THREADS threads x CT_PER cells
constexpr int CT_THREADS = 256, CT_PER = 16;
constexpr int AGG_STRIDE = WL_CLASSES + 1;   // [0, WL_CLASSES): cells per class, [WL_CLASSES]: kept points

// 16 consecutive cells per thread: eight 16-byte loads of the (runs << 32 | points) counters; c = points, r (optional) = runs
__device__ __forceinline__ void load_tile_counts(const unsigned long long* cnt64, int N2, int cell0, int c[CT_PER], int* r = nullptr) {
    if (cell0 + CT_PER <= N2 && (((size_t)cnt64 & 15) == 0) && (cell0 & 1) == 0) {
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(cnt64 + cell0);
#pragma unroll
        for (int q = 0; q < CT_PER / 2; ++q) {
            const ulonglong2 v = p[q];
            c[2 * q] = (int)(uint32_t)v.x;
            c[2 * q + 1] = (int)(uint32_t)v.y;
            if (r) {
                r[2 * q] = (int)(v.x >> 32);
                r[2 * q + 1] = (int)(v.y >> 32);
            }
        }
    } else {
#pragma unroll
        for (int q = 0; q < CT_PER; ++q) {
            const unsigned long long v = (cell0 + q < N2) ? cnt64[cell0 + q] : 0ull;
            c[q] = (int)(uint32_t)v;
            if (r) r[q] = (int)(v >> 32);
        }
    }
}

__global__ void __launch_bounds__(CT_THREADS) k_cell_tiles(View v, const SlotParams* __restrict__ batch) {
    __shared__ int s_cls[AGG_STRIDE];
    const SlotParams& sp = batch[blockIdx.y];
    const int N2 = v.k.N2, tid = threadIdx.x, lane = tid & 31;
    if (tid < AGG_STRIDE) s_cls[tid] = 0;
    __syncthreads();
    int c[CT_PER];
    load_tile_counts(v.cnt64 + (size_t)sp.slot * N2, N2, blockIdx.x * CELL_TILE + tid * CT_PER, c);
    int sum = 0;
#pragma unroll
    for (int q = 0; q < CT_PER; ++q) {
        sum += c[q];
        if (c[q] > 0) atomicAdd(&s_cls[worklist_class(c[q])], 1);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
    if (lane == 0 && sum) atomicAdd(&s_cls[WL_CLASSES], sum);
    __syncthreads();
    if (tid < AGG_STRIDE) v.cell_agg[((size_t)sp.slot * v.cell_tiles + blockIdx.x) * AGG_STRIDE + tid] = s_cls[tid];
}

__global__ void __launch_bounds__(CT_THREADS) k_cell_place(View v, const SlotParams* __restrict__ batch) {
    __shared__ int s_cur[AGG_STRIDE];   // worklist cursor of every class for this tile; [WL_CLASSES]: first segment start of the tile
    __shared__ int s_warp[CT_THREADS / 32];
    const SlotParams& sp = batch[blockIdx.y];
    const int N2 = v.k.N2, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tiles = v.cell_tiles, tile = blockIdx.x;
    const int* agg = v.cell_agg + (size_t)sp.slot * tiles * AGG_STRIDE;
    const size_t off = (size_t)sp.slot * N2;
    const int cell0 = tile * CELL_TILE + tid * CT_PER;
    int c[CT_PER], rn[CT_PER];
    load_tile_counts(v.cnt64 + off, N2, cell0, c, rn);
    // one warp: per class (2 per lane) the total over all tiles and the part of the earlier tiles
    if (warp == 0) {
        int tot[2] = {0, 0}, pre[2] = {0, 0};
        const int k0 = WL_CLASSES - 1 - 2 * lane, k1 = k0 - 1;   // lane 0: classes 63, 62 ... lane 31: classes 1, 0
        for (int p = 0; p < tiles; ++p) {
            const int a0 = agg[p * AGG_STRIDE + k0], a1 = agg[p * AGG_STRIDE + k1];
            tot[0] += a0;
            tot[1] += a1;
            if (p < tile) {
                pre[0] += a0;
                pre[1] += a1;
            }
        }
        const int incl = warp_inclusive_scan(tot[0] + tot[1]);   // classes in descending order: heaviest first
        s_cur[k0] = incl - tot[0] - tot[1] + pre[0];
        s_cur[k1] = incl - tot[1] + pre[1];
        int pts = 0, pts_all = 0;
        for (int p = lane; p < tiles; p += 32) {
            const int a = agg[p * AGG_STRIDE + WL_CLASSES];
            pts_all += a;
            if (p < tile) pts += a;
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            pts += __shfl_xor_sync(0xffffffffu, pts, d);
            pts_all += __shfl_xor_sync(0xffffffffu, pts_all, d);
        }
        if (lane == 0) s_cur[WL_CLASSES] = pts;
        if (tile == 0 && lane == 31) {
            v.wl_count[2 * sp.slot] = incl;          // non-empty cells of the scan
            v.wl_count[2 * sp.slot + 1] = pts_all;   // kept points of the scan (= end of the last segment)
        }
    }
    int sum = 0;
#pragma unroll
    for (int q = 0; q < CT_PER; ++q) sum += c[q];
    const int incl = warp_inclusive_scan(sum);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int run = s_cur[WL_CLASSES] + incl - sum;
    for (int w = 0; w < warp; ++w) run += s_warp[w];
    // a worklist entry carries everything k_cell_stats needs to start on the cell: (cell, points, runs, segment start)
    int4* wl = v.worklist + off;
    int cs[CT_PER];
#pragma unroll
    for (int q = 0; q < CT_PER; ++q) {
        cs[q] = run;
        if (c[q] > 0) wl[atomicAdd(&s_cur[worklist_class(c[q])], 1)] = make_int4(cell0 + q, c[q], rn[q], run);
        run += c[q];
    }
    if (cell0 + CT_PER <= N2 && (N2 & 3) == 0) {
        int4* dst = reinterpret_cast<int4*>(v.cellstart + off + cell0);
#pragma unroll
        for (int q = 0; q < CT_PER / 4; ++q) dst[q] = make_int4(cs[4 * q], cs[4 * q + 1], cs[4 * q + 2], cs[4 * q + 3]);
    } else {
#pragma unroll
        for (int q = 0; q < CT_PER; ++q)
            if (cell0 + q < N2) v.cellstart[off + cell0 + q] = cs[q];
    }
}

constexpr int SCATTER_ILP = 4;

// Directory entry of a run, at rundir[cellstart + arrival number] (a cell has at most as many runs as points):
//   x = run id (point index >> 5), y = first position inside the segment | (length - 1) << 26
__global__ void __launch_bounds__(256) k_scatter(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.y];
    const int n = sp.n_points;
    const int i0 = blockIdx.x * (256 * SCATTER_ILP) + threadIdx.x;
    if (i0 >= n) return;
    const size_t base = (size_t)sp.slot * v.pcap;
    const int* cellstart = v.cellstart + (size_t)sp.slot * v.k.N2;
    float* zs = v.zsorted + base;
    uint2* dir = v.rundir + base;
    uint32_t code[SCATTER_ILP];
    uint2 zw[SCATTER_ILP];
    int cs[SCATTER_ILP];
    uint32_t jl[SCATTER_ILP];
#pragma unroll
    for (int u = 0; u < SCATTER_ILP; ++u) {
        const int i = i0 + u * 256;
        code[u] = i < n ? v.code[base + i] : (PC_ABSENT << 24);
        zw[u] = i < n ? v.zw[base + i] : make_uint2(0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < SCATTER_ILP; ++u) {
        const uint32_t cls = code[u] >> 24;
        const bool kept = cls == PC_KEPT || cls == PC_KEPT_BORDER;
        cs[u] = kept ? cellstart[code[u] & 0xffffffu] : -1;
        jl[u] = (kept && (zw[u].y & 0x80000000u)) ? v.runj[base + i0 + u * 256] : 0u;
    }
#pragma unroll
    for (int u = 0; u < SCATTER_ILP; ++u) {
        if (cs[u] < 0) continue;
        const uint32_t p = zw[u].y & 0x7fffffffu;
        zs[cs[u] + (int)p] = __uint_as_float(zw[u].x);
        if (zw[u].y & 0x80000000u) dir[cs[u] + (int)(jl[u] & RUN_LOW26)] = make_uint2((uint32_t)((i0 + u * 256) >> 5), p | (jl[u] & ~RUN_LOW26));
    }
}

// ------------------------------------------------------------------------------------------
// phase 1c: per-cell sequential statistics (the accumulate step of insert_cloud, :282-309,
// in input order) + variance (:323).  One thread per cell.
// ------------------------------------------------------------------------------------------
constexpr int CS_THREADS = 256;

// "pointsRaw" of a cell with r inside points.  The reference counts up by 1.0f (:234), which stops at 2^24 (2^24 + 1
// rounds back to 2^24); raw_i counts in int, so the float it stores is clamped to where the float count stops.
__device__ __forceinline__ float raw_count(int r) { return (float)min(r, 1 << 24); }

template <bool FULL>
__global__ void __launch_bounds__(CS_THREADS, FULL ? 2 : 4) k_cell_stats(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.y];
    const Const& k = v.k;
    const size_t coff = (size_t)sp.slot * k.N2;
    const int gt = blockIdx.x * CS_THREADS + threadIdx.x;
    const int kept_total = v.wl_count[2 * sp.slot + 1];
    // (1) four consecutive cells per thread, coalesced: the per-scan resets every cell needs, and the results of an
    //     EMPTY cell (count 0, m2 / (0 + FLT_MIN) = 0, min = FLT_MAX, :61-75,323).  Empty <=> zero-length segment
    //     (the counters themselves are being consumed by other threads of this launch).
    for (int t = gt * 4; t < k.N2; t += gridDim.x * CS_THREADS * 4) {
        int cs[5];
#pragma unroll
        for (int q = 0; q < 5; ++q) cs[q] = (t + q < k.N2) ? v.cellstart[coff + t + q] : kept_total;
        if ((k.N2 & 3) == 0) {
            *reinterpret_cast<float4*>(v.layer(sp.slot, L_OBSTACLES) + t) = make_float4(0.f, 0.f, 0.f, 0.f);  // map["points"].setConstant(0.0), :147
            if (FULL) {
                const int4 r = *reinterpret_cast<const int4*>(v.raw_i + coff + t);
                *reinterpret_cast<float4*>(v.layer(sp.slot, L_RAW) + t) = make_float4(raw_count(r.x), raw_count(r.y), raw_count(r.z), raw_count(r.w));
                *reinterpret_cast<int4*>(v.raw_i + coff + t) = make_int4(0, 0, 0, 0);
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int cell = t + q;
            if (cell >= k.N2) break;
            if ((k.N2 & 3) != 0) {
                v.layer(sp.slot, L_OBSTACLES)[cell] = 0.0f;
                if (FULL) {
                    v.layer(sp.slot, L_RAW)[cell] = raw_count(v.raw_i[coff + cell]);
                    v.raw_i[coff + cell] = 0;
                }
            }
            if (cs[q + 1] == cs[q]) {
                v.layer(sp.slot, L_COUNT)[cell] = 0.0f;
                v.layer(sp.slot, L_VARIANCE)[cell] = 0.0f;
                v.layer(sp.slot, L_MINH)[cell] = FLT_MAX;
                if (FULL) {
                    v.layer(sp.slot, L_M2)[cell] = 0.0f;
                    v.layer(sp.slot, L_MEAN)[cell] = 0.0f;
                    v.layer(sp.slot, L_GCAND)[cell] = 0.0f;
                    v.layer(sp.slot, L_PLANEDIST)[cell] = 0.0f;
                    v.layer(sp.slot, L_MAXH)[cell] = FLT_MIN;
                }
            }
        }
    }
    // (2) the worklist: non-empty cells grouped by count class (k_cell_place), so the 32 cells of a warp need (almost)
    //     the same number of sequential steps; grid-stride (a warp's entries stay 32 consecutive ones)
    const int wl_n = v.wl_count[2 * sp.slot];
    const float oz = sp.oz;
    for (int t = gt; t < wl_n; t += gridDim.x * CS_THREADS) {
    const int4 entry = v.worklist[coff + t];   // one load instead of a chain of three dependent ones
    const int cell = entry.x, cnt = entry.y, runs = entry.z, cstart = entry.w;
    const float* zs = v.zsorted + (size_t)sp.slot * v.pcap + cstart;
    uint2* dir = v.rundir + (size_t)sp.slot * v.pcap + cstart;
    // the kernel is bound by the latency of dependent global loads: pull the first lines of the segment and of the
    // run directory towards L1 right away
    asm volatile("prefetch.global.L1 [%0];" ::"l"(zs));
    if (cnt > 32) asm volatile("prefetch.global.L1 [%0];" ::"l"(zs + 32));
    if (runs > 1) asm volatile("prefetch.global.L1 [%0];" ::"l"(dir));

    float n = 0.0f, mean = 0.0f, m2 = 0.0f;
    float mn = FLT_MAX;
    float mx = FLT_MIN, gc = 0.0f, pdm = 0.0f;  // dead layers (FULL only)
    // one accumulate step of insert_cloud (:282-309)
    auto step = [&](float z) {
        const float pd = __fsub_rn(z, oz);  // planeDist, :295
        if (FULL) gc = (float)__ddiv_rn((double)__fadd_rn(z, __fmul_rn(n, gc)), __dadd_rn((double)n, 1.0));  // :296
        if (mean == 0.0f) mean = pd;  // :298-299
        if (!(pd != pd)) {            // :300
            const float delta = __fsub_rn(pd, mean);
            mean = __fadd_rn(mean, __fdiv_rn(delta, __fadd_rn(n, 1.0f)));
            if (FULL) pdm = (float)__ddiv_rn((double)__fadd_rn(pd, __fmul_rn(n, pdm)), __dadd_rn((double)n, 1.0));
            m2 = __fadd_rn(m2, __fmul_rn(delta, __fsub_rn(pd, mean)));
        }
        if (FULL) mx = (mx < z) ? z : mx;                   // std::max(maxHeight, z)
        const float zl = __fsub_rn(z, 0.0001f);
        mn = (zl < mn) ? zl : mn;                           // std::min(minHeight, z - 0.0001f)
        n = __fadd_rn(n, 1.0f);
    };

    // The segment is a sequence of runs (k_rasterize), each internally in input order; input order of the cell = runs
    // by ascending id.  The cell's directory (one entry per run, contiguous) is sorted by id first: up to 8 runs in
    // registers (odd-even transposition), more -- cells crossed by many rings: walls, vehicles -- by an in-place Shell
    // sort (gaps 57 / 23 / 10 / 4 / 1).
    if (runs > 1 && runs <= 8) {
        uint2 e[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) e[q] = (q < runs) ? dir[q] : make_uint2(0xffffffffu, 0u);
        bool moved = false;
#pragma unroll
        for (int pass = 0; pass < 8; ++pass) {
#pragma unroll
            for (int q = pass & 1; q + 1 < 8; q += 2) {
                if (e[q + 1].x < e[q].x) {
                    const uint2 tmp = e[q];
                    e[q] = e[q + 1];
                    e[q + 1] = tmp;
                    moved = true;
                }
            }
        }
        if (moved) {
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (q < runs) dir[q] = e[q];
        }
    } else if (runs > 8) {
        const int gaps[5] = {57, 23, 10, 4, 1};
#pragma unroll
        for (int gi = 0; gi < 5; ++gi) {
            const int gap = gaps[gi];
            if (gap >= runs) continue;
            for (int a = gap; a < runs; ++a) {
                const uint2 e = dir[a];
                int b = a;
                while (b >= gap) {
                    const uint2 f = dir[b - gap];
                    if (f.x <= e.x) break;
                    dir[b] = f;
                    b -= gap;
                }
                if (b != a) dir[b] = e;
            }
        }
    }
    // Streaming walk: chunks of up to 8 consecutive heights of the current run; the loads of the next chunk (and the
    // directory entry of the next run) are in flight while the current chunk goes through the sequential recurrence.
    {
        int rj = 0, pb = 0, pe = cnt;   // runs == 1: the whole segment
        if (runs > 1) {
            const uint2 e0 = dir[0];
            pb = (int)(e0.y & RUN_LOW26);
            pe = pb + (int)(e0.y >> 26) + 1;
        }
        float zb[8], zn[8];
        int mb = 0, mnx = 0;
        auto fetch = [&](float* dst, int& m) {
            m = min(8, pe - pb);
#pragma unroll
            for (int q = 0; q < 8; ++q) dst[q] = (q < m) ? zs[pb + q] : 0.0f;
            pb += m;
            if (pb == pe && ++rj < runs) {
                const uint2 en = dir[rj];
                pb = (int)(en.y & RUN_LOW26);
                pe = pb + (int)(en.y >> 26) + 1;
                if (((pb + 8) & ~31) != (pb & ~31)) asm volatile("prefetch.global.L1 [%0];" ::"l"(zs + pb + 8));
            }
        };
        fetch(zb, mb);
        while (mb > 0) {
            fetch(zn, mnx);
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (q < mb) step(zb[q]);
#pragma unroll
            for (int q = 0; q < 8; ++q) zb[q] = zn[q];
            mb = mnx;
        }
    }
    v.cnt64[coff + cell] = 0ull;                   // consumed: zero again for the next scan
    v.layer(sp.slot, L_COUNT)[cell] = n;
    v.layer(sp.slot, L_VARIANCE)[cell] = __fdiv_rn(m2, __fadd_rn(n, FLT_MIN));
    v.layer(sp.slot, L_MINH)[cell] = mn;
    if (FULL) {
        v.layer(sp.slot, L_M2)[cell] = m2;
        v.layer(sp.slot, L_MEAN)[cell] = mean;
        v.layer(sp.slot, L_GCAND)[cell] = gc;
        v.layer(sp.slot, L_PLANEDIST)[cell] = pdm;
        v.layer(sp.slot, L_MAXH)[cell] = mx;
    }
    }
}

// ------------------------------------------------------------------------------------------
// phase 2: ground patch detection stencil (detect_ground_patches / detect_ground_patch<S>)
// ------------------------------------------------------------------------------------------
constexpr int DT_X = 32, DT_Y = 8, DT_H = 2;
constexpr int DT_W = DT_X + 2 * DT_H;   // 36
constexpr int DT_R = DT_Y + 2 * DT_H;   // 12

// the confidence decay of interpolate_cell (:464) is gg_internal.h:decay_confidence

// Fused into k_detect: every cell is copied to its home slot(s) as soon as its final G, C are known.
__device__ __forceinline__ void skew_store_cell(const View& v, const SlotParams& sp, int cell, int x, int y, float g, float c, bool far) {
    const Const& k = v.k;
    const CfgConst& kc = sp.cfg;
    const int4 home = __ldg(reinterpret_cast<const int4*>(v.skew.cell_home) + cell);
    if (home.x < 0) return;
    const int cidx = k.N / 2 - 1;
    if (x == cidx && y == cidx) {  // spiral_ground_interpolation :405,411 (the normal layers get it in k_spiral_skew)
        g = sp.base_z_f;
        c = 1.0f;
    }
    // :463: beyond minDistSquared (`far`, from the per-cell table) the visit stores the decayed confidence (:464)
    const float d1 = far ? decay_confidence(kc, c) : SKEW_NEAR;
    float2* SK = v.skew.sk + (size_t)sp.slot * v.skew.slots;
    float* SD = v.skew.sd + (size_t)sp.slot * v.skew.slots;
    const float2 gc = make_float2(g, c);
    SK[home.x] = gc;
    SD[home.x] = d1;
    if (home.y >= 0) {
        SK[home.y] = gc;
        SD[home.y] = far ? decay_confidence(kc, d1) : SKEW_NEAR;  // second visit of a ring corner
    }
    if (home.z >= 0) SK[home.z] = gc;
    if (home.w >= 0) SK[home.w] = gc;
}

// Per-cell quantities of detect_ground_patches that depend only on the grid and the configuration, computed
// once per configuration variant (gg_capi.cu:build_variant) with the very operations of the per-scan code they replace:
//   x: max(3, floor(threshold * S * expectedPoints))  (:364), rounded up to float: for a float psum, psum < x is then the
//      reference's double comparison psum < max(...) at any magnitude (no float lies between the bound and x)
//   y: variance threshold (:369)      z: expectedPoints      w: flags
constexpr int DTF_S5 = 1, DTF_FAR = 2, DTF_INNER = 4;

__global__ void k_build_detect_table(View v, const CfgConst kc, float4* __restrict__ tab) {
    const Const& k = v.k;
    const int N = k.N;
    const int cell = blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= k.N2) return;
    const int i = cell % N, j = cell / N;
    const double di = __dsub_rn((double)i, (double)N / 2.0), dj = __dsub_rn((double)j, (double)N / 2.0);
    const float sqdist = (float)__dmul_rn(__dadd_rn(__dmul_rn(di, di), __dmul_rn(dj, dj)), k.res_sq);  // :332,356
    const float e = v.expected[cell];
    int flags = 0;
    if (!((double)sqdist <= kc.psc_sq)) flags |= DTF_S5;
    // union of the four sections, :325-328: first index in [2, 2 * (N / 2) - 2) (the upper half starts at N / 2 and has
    // N / 2 - 2 entries: one row short of N - 2 when N is odd), second index in [2, N - 2)
    if (i >= 2 && i < 2 * (N / 2) - 2 && j >= 2 && j < N - 2) flags |= DTF_INNER;
    const int cidx = N / 2 - 1;
    const float fx = __fsub_rn((float)i, (float)cidx), fy = __fsub_rn((float)j, (float)cidx);
    if (__dmul_rn(__dadd_rn(__dmul_rn((double)fx, (double)fx), __dmul_rn((double)fy, (double)fy)), k.res_sq) > 12.0) flags |= DTF_FAR;  // :463
    const double S = (flags & DTF_S5) ? 5.0 : 3.0;
    double need = floor(__dmul_rn(__dmul_rn(kc.gp_thresh, S), (double)e));
    need = (need < 3.0) ? 3.0 : need;                 // NaN -> NaN: the comparison below stays false, as in the reference
    const double a = __dmul_rn((double)sqdist, kc.df_sq);
    const double m = (a < kc.mdf_sq) ? kc.mdf_sq : a;
    const float vt = (float)((kc.mdf10_sq < m) ? kc.mdf10_sq : m);
    tab[cell] = make_float4(__double2float_ru(need), vt, e, __int_as_float(flags));
}

// returns true when (g, c) changed
// sPV / sPM hold the products count * variance and count * minHeight of every tile entry (the very fmul the
// reference's cwiseProduct performs, done once per entry instead of once per window position)
template <int S>
__device__ __forceinline__ bool detect_patch(const CfgConst& kc, const float (*sP)[DT_W], const float (*sPV)[DT_W], const float (*sPM)[DT_W],
                                             const float (*sM)[DT_W], int li, int lj, float variance, float need, float vt, float e, float& g,
                                             float& c) {
    constexpr int H = S / 2;
    const int r0 = li - H, c0 = lj - H;  // block origin in the shared tile (row index = i, col = j)
    const float psum = TreeSum<0, S * S>::run([&](int q) { return sP[c0 + q / S][r0 + q % S]; });
    const float oc = c, og = g;

    // early skipping of (almost) empty areas, :364 (need is rounded up to float: the float compare is the double one)
    if (psum < need) return false;

    float localmin = sM[c0][r0];
#pragma unroll
    for (int q = 1; q < S * S; ++q) {
        const float t = sM[c0 + q / S][r0 + q % S];
        localmin = (t < localmin) ? t : localmin;
    }
    const float maxVar = (sP[lj][li] >= kc.pc_var_thresh_f)
                             ? variance
                             : __fdiv_rn(TreeSum<0, S * S>::run([&](int q) { return sPV[c0 + q / S][r0 + q % S]; }), psum);
    const float groundlevel = __fdiv_rn(TreeSum<0, S * S>::run([&](int q) { return sPM[c0 + q / S][r0 + q % S]; }), psum);
    const float gd = __fmul_rn(__fsub_rn(groundlevel, og), __fmul_rn(2.0f, oc));
    const float groundDiff = (gd < 1.0f) ? 1.0f : gd;  // std::max(gd, 1.0f)

    // do not update known high confidence estimations upward, :379
    if ((double)oc > 0.5 && (double)groundlevel >= __dadd_rn((double)og, kc.outlier_tol)) return false;

    if ((double)vt > __dmul_rn((double)maxVar, (double)maxVar) && maxVar > 0.0f &&
        (double)psum > __dmul_rn((double)__fmul_rn(__fmul_rn(groundDiff, e), (float)S), kc.gp_thresh)) {
        const double ncd = __ddiv_rn((double)psum, kc.occ_factor);
        const float nc = (float)((1.0 < ncd) ? 1.0 : ncd);  // std::min(ncd, 1.0)
        const float num = __fadd_rn(__fmul_rn(groundlevel, nc), __fmul_rn(__fmul_rn(oc, og), 2.0f));
        const float den = __fadd_rn(nc, __fmul_rn(oc, 2.0f));
        g = __fdiv_rn(num, den);
        const double cd = __ddiv_rn(__dadd_rn(__ddiv_rn((double)psum, kc.occ_factor2), (double)oc), 2.0);
        c = (float)((1.0 < cd) ? 1.0 : cd);
        return true;
    }
    if (localmin < og) {
        g = localmin;
        const float t = __fadd_rn(oc, 0.1f);
        c = (0.5f < t) ? 0.5f : t;  // std::min(oc + 0.1f, 0.5f)
        return true;
    }
    return false;
}

// count_layer: the plane read as "points" -- L_COUNT in the pipeline, whatever "points" names for a call on its own.
// recompute (a call on its own, full layers): the variance is m2 / (points + FLT_MIN) (:323), computed from L_M2 for
// every tile entry and stored for every cell, instead of read from L_VARIANCE (the pipeline's k_cell_stats just wrote it).
__global__ void __launch_bounds__(DT_X* DT_Y, 5) k_detect_ldg(View v, const SlotParams* __restrict__ batch, int count_layer, bool recompute) {
    __shared__ float sP[DT_R][DT_W], sPV[DT_R][DT_W], sPM[DT_R][DT_W], sM[DT_R][DT_W];
    const SlotParams& sp = batch[blockIdx.z];
    const Const& k = v.k;
    const CfgConst& kc = sp.cfg;
    const int N = k.N;
    const int i0 = blockIdx.x * DT_X, j0 = blockIdx.y * DT_Y;
    // one 64-bit base per scan, 32-bit offsets below it (all layers of a slot span far less than 2^31 floats)
    float* const L0 = v.layer(sp.slot, 0);
    const int N2 = k.N2;
    const float* P = L0 + count_layer * N2;
    const float* V = L0 + (recompute ? L_M2 : L_VARIANCE) * N2;
    const float* M = L0 + L_MINH * N2;
    // tile + halo (36 x 12): a thread fetches column tx of rows ty and ty + 8 (ty < 4) and, for tx < 4, the halo
    // columns 32 + tx of the same rows; four fixed positions o, o + 32, o + 8 N, o + 8 N + 32, every global load issued
    // before the first shared store.  Outside the map: count 0, variance 0, min FLT_MAX (products 0), as before.
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int gi = i0 - DT_H + tx, gj = j0 - DT_H + ty;
    const bool col0 = gi >= 0 && gi < N, col1 = tx < 2 * DT_H && gi + DT_X < N;
    const bool row0 = gj >= 0 && gj < N, row1 = ty < 2 * DT_H && gj + DT_Y < N;
    const int o = gi + gj * N;
    const bool in[4] = {col0 && row0, col1 && row0, col0 && row1, col1 && row1};
    const int off[4] = {o, o + DT_X, o + DT_Y * N, o + DT_Y * N + DT_X};
    float tp[4], tv[4], tm[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        tp[u] = in[u] ? P[off[u]] : 0.0f;
        tv[u] = in[u] ? V[off[u]] : 0.0f;
        tm[u] = in[u] ? M[off[u]] : FLT_MAX;
        if (recompute) tv[u] = __fdiv_rn(tv[u], __fadd_rn(tp[u], FLT_MIN));   // outside the map 0 / FLT_MIN = 0, as before
    }
    const int i = i0 + tx, j = j0 + ty;
    const bool live = i < N && j < N;
    const int cell = i + j * N;
    float g = 0.0f, c = 0.0f, variance = 0.0f;
    float4 tb = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (live) {
        g = L0[L_GROUND * N2 + cell];
        c = L0[L_GROUNDPATCH * N2 + cell];
        variance = V[cell];
        tb = __ldg(sp.detect_tab + cell);
        if (recompute) {
            variance = __fdiv_rn(variance, __fadd_rn(P[cell], FLT_MIN));
            L0[L_VARIANCE * N2 + cell] = variance;   // no block reads L_VARIANCE in this mode
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const bool mine = ((u & 1) == 0 || tx < 2 * DT_H) && ((u & 2) == 0 || ty < 2 * DT_H);
        if (mine) {
            const int li = (u & 1) ? DT_X + tx : tx, lj = (u & 2) ? ty + DT_Y : ty;
            sP[lj][li] = tp[u];
            sPV[lj][li] = __fmul_rn(tp[u], tv[u]);
            sPM[lj][li] = __fmul_rn(tp[u], tm[u]);
            sM[lj][li] = tm[u];
        }
    }
    __syncthreads();
    if (!live) return;
    const int flags = __float_as_int(tb.w);
    if (flags & DTF_INNER) {
        const int li = threadIdx.x + DT_H, lj = threadIdx.y + DT_H;
        const bool changed = (flags & DTF_S5) ? detect_patch<5>(kc, sP, sPV, sPM, sM, li, lj, variance, tb.x, tb.y, tb.z, g, c)
                                              : detect_patch<3>(kc, sP, sPV, sPM, sM, li, lj, variance, tb.x, tb.y, tb.z, g, c);
        if (changed) {
            L0[L_GROUND * N2 + cell] = g;
            L0[L_GROUNDPATCH * N2 + cell] = c;
        }
    }
    if (v.skew.sk) {
        skew_store_cell(v, sp, cell, i, j, g, c, (flags & DTF_FAR) != 0);
    } else if (v.spiral_recs) {
        // Decayed confidence for the spiral sweep, taken off its sequential critical path: the
        // confidence of a cell only changes at its own visit(s), so decay(C) after patch
        // detection is exactly what the (first) visit will store; ring corners (i == j) are
        // visited twice and need the second decay as well.
        const float d1 = decay_confidence(kc, c);
        float* D1 = v.roll_scratch + (size_t)sp.slot * 2 * k.N2;
        D1[cell] = d1;
        if (i == j) D1[k.N2 + cell] = decay_confidence(kc, d1);
    }
}

// ---- TMA-staged variant ------------------------------------------------------------------
// The tile (+halo) of the three per-scan layers arrives by three cp.async.bulk.tensor loads (one elected thread, one
// mbarrier); cells outside the map are zero-filled by the TMA unit, which is harmless because only cells [2, N-2)
// compute and their windows stay inside the map (:325-337).  The innermost start coordinate of a TMA box must be
// 16-byte aligned (a start at i0 - 2 is not a valid TMA box origin), so the
// tile keeps a halo of 4 cells in i: box = 40 x 12 x 1 at (i0 - 4, j0 - 2).  All layers of all slots form ONE 3-D tensor
// (i, j, plane = slot * n_layers + layer), so one descriptor serves every scan.  While the tile is in flight the
// threads fetch their own cell's G, C and table entry.
//
// Window sums.  The three block reductions of :359,374-375 are Eigen's binary-split tree over the column-major
// coefficients e[k] = block(k % S, k / S) (SURVEY App. A.0).  Most inner nodes of that tree are runs of 2 or 3
// consecutive rows of ONE column: pair(r, c) = q(r, c) + q(r+1, c) and triple(r, c) = q(r, c) + pair(r+1, c) -- the
// very additions of the tree, so they can be computed once per tile position and shared by every window that contains
// them (a 5x5 tree then needs 14 shared loads and 13 additions instead of 25 and 24).  The point-count sum is taken
// from column partials of 3 / 5 rows: exact in any order while every count of the tile is an integer in
// [0, DT_EXACT_COUNT] (25 of them stay below 2^24); a tile holding any other count (an imported plane: fractions,
// negatives, NaN, huge counts) sums every window in Eigen's tree order instead.  The block minimum is taken from
// column minima that skip NaN, then across the columns, and is the NaN of element 0 when there is one: the minCoeff
// fold keeps its first element unless a later one is strictly smaller, so a NaN elsewhere never counts.  Tiles
// without a single candidate cell (psum >= need nowhere) skip the product stage.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}

constexpr int DT_HX = 4;                 // halo in i of the TMA tile (alignment of the box start)
constexpr int DT_WT = DT_X + 2 * DT_HX;  // 40
constexpr int DT_WC = DT_WT - 4;         // 36: columns that can be the first row of a 3 / 5-row window
constexpr int DT_WB = DT_WT - 2;         // 38: columns whose product is read by some window

struct __align__(128) DetectRaw {   // one pipeline stage: the three TMA destinations
    float P[DT_R][DT_WT];   // kept points per cell
    float V[DT_R][DT_WT];   // variance
    float M[DT_R][DT_WT];   // min height
};
struct __align__(128) DetectTile {
    DetectRaw raw[2];       // double buffer: the tile after next is in flight while this one is computed
    float C3[DT_R][DT_WT], C5[DT_R][DT_WT];       // sum of P over rows r .. r+2 / r .. r+4 of the column (exact integers)
    float N3[DT_R][DT_WT], N5[DT_R][DT_WT];       // min of M over the same rows
    float QV[DT_R][DT_WT], PV2[DT_R][DT_WT], TV[DT_R][DT_WT];   // q = P * V; pair; triple
    float QM[DT_R][DT_WT], PM2[DT_R][DT_WT], TM[DT_R][DT_WT];   // q = P * M; pair; triple
};
static_assert(offsetof(DetectRaw, V) % 128 == 0 && offsetof(DetectRaw, M) % 128 == 0 && sizeof(DetectRaw) % 128 == 0, "TMA destinations are 128-byte aligned");   // 12 * 40 * 4 = 1920 = 15 * 128

// Eigen tree of a 5x5 / 3x3 window from the shared partials; (r0, c0) = window origin (row = i, col = j)
__device__ __forceinline__ float tree25(const float (*Q)[DT_WT], const float (*P2)[DT_WT], const float (*T)[DT_WT], int r0, int c0) {
#define QQ(r, c) Q[c0 + (c)][r0 + (r)]
#define PP(r, c) P2[c0 + (c)][r0 + (r)]
#define TT(r, c) T[c0 + (c)][r0 + (r)]
    const float s0_6 = __fadd_rn(TT(0, 0), __fadd_rn(QQ(3, 0), __fadd_rn(QQ(4, 0), QQ(0, 1))));          // e0..e2 | e3 + (e4 + e5)
    const float s6_6 = __fadd_rn(TT(1, 1), __fadd_rn(QQ(4, 1), PP(0, 2)));                                  // e6..e8 | e9 + (e10 + e11)
    const float s12_6 = __fadd_rn(TT(2, 2), TT(0, 3));                                                      // e12..e14 | e15..e17
    const float s18_7 = __fadd_rn(__fadd_rn(QQ(3, 3), __fadd_rn(QQ(4, 3), QQ(0, 4))), __fadd_rn(PP(1, 4), PP(3, 4)));  // e18 + (e19 + e20) | (e21 + e22) + (e23 + e24)
    return __fadd_rn(__fadd_rn(s0_6, s6_6), __fadd_rn(s12_6, s18_7));
#undef TT
}
__device__ __forceinline__ float tree9s(const float (*Q)[DT_WT], const float (*P2)[DT_WT], int r0, int c0) {
    const float s0_4 = __fadd_rn(PP(0, 0), __fadd_rn(QQ(2, 0), QQ(0, 1)));                  // (e0 + e1) + (e2 + e3)
    const float s4_5 = __fadd_rn(PP(1, 1), __fadd_rn(QQ(0, 2), PP(1, 2)));                  // (e4 + e5) + (e6 + (e7 + e8))
    return __fadd_rn(s0_4, s4_5);
#undef QQ
#undef PP
}

// the decision part of detect_ground_patch<S> (:364-394) on the window quantities; returns true when (g, c) changed
template <int S>
__device__ __forceinline__ bool detect_decide(const CfgConst& kc, float psum, float localmin, float sumPV, float sumPM, float centerP, float variance, float vt,
                                              float e, float& g, float& c) {
    const float oc = c, og = g;
    const float maxVar = (centerP >= kc.pc_var_thresh_f) ? variance : __fdiv_rn(sumPV, psum);
    const float groundlevel = __fdiv_rn(sumPM, psum);
    const float gd = __fmul_rn(__fsub_rn(groundlevel, og), __fmul_rn(2.0f, oc));
    const float groundDiff = (gd < 1.0f) ? 1.0f : gd;  // std::max(gd, 1.0f)
    // do not update known high confidence estimations upward, :379
    if ((double)oc > 0.5 && (double)groundlevel >= __dadd_rn((double)og, kc.outlier_tol)) return false;
    if ((double)vt > __dmul_rn((double)maxVar, (double)maxVar) && maxVar > 0.0f &&
        (double)psum > __dmul_rn((double)__fmul_rn(__fmul_rn(groundDiff, e), (float)S), kc.gp_thresh)) {
        // std::min(psum / factor, 1.0): a quotient of at least one needs no division (psum >= factor > 0 <=> quotient >= 1)
        float nc = 1.0f;
        if (!(kc.occ_factor > 0.0 && (double)psum >= kc.occ_factor)) {
            const double ncd = __ddiv_rn((double)psum, kc.occ_factor);
            nc = (float)((1.0 < ncd) ? 1.0 : ncd);
        }
        const float num = __fadd_rn(__fmul_rn(groundlevel, nc), __fmul_rn(__fmul_rn(oc, og), 2.0f));
        const float den = __fadd_rn(nc, __fmul_rn(oc, 2.0f));
        g = __fdiv_rn(num, den);
        // std::min((psum / (factor * 2.0f) + oc) / 2.0, 1.0): halving is exact (x * 0.5)
        const double cd = __dmul_rn(__dadd_rn(__ddiv_rn((double)psum, kc.occ_factor2), (double)oc), 0.5);
        c = (float)((1.0 < cd) ? 1.0 : cd);
        return true;
    }
    if (localmin < og) {
        g = localmin;
        const float t = __fadd_rn(oc, 0.1f);
        c = (0.5f < t) ? 0.5f : t;  // std::min(oc + 0.1f, 0.5f)
        return true;
    }
    return false;
}

// A CTA walks DT_TILES consecutive tiles along j; the TMA loads of tile k + 1 are issued before tile k is computed
// (two stages of raw tiles, one mbarrier each, phase parity flips every second use).
constexpr int DT_TILES = 4;
constexpr float DT_EXACT_COUNT = 524288.0f;   // 2^19: 25 such counts sum to less than 2^24

// the minimum of a, b that keeps a unless b is strictly smaller, or a is NaN (column minima that skip NaN)
__device__ __forceinline__ float min_skip_nan(float a, float b) { return (b < a || a != a) ? b : a; }

__global__ void __launch_bounds__(DT_X* DT_Y, 5) k_detect_tma(View v, const SlotParams* __restrict__ batch, const __grid_constant__ CUtensorMap tmap,
                                                             int count_layer, bool recompute) {
    __shared__ DetectTile s;
    __shared__ __align__(8) uint64_t s_bar[2];
    const SlotParams& sp = batch[blockIdx.z];
    const Const& k = v.k;
    const CfgConst& kc = sp.cfg;
    const int N = k.N, N2 = k.N2;
    const int i0 = blockIdx.x * DT_X;
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * DT_X + tx;
    const int tile0 = blockIdx.y * DT_TILES;
    const int n_tiles = min(DT_TILES, (N + DT_Y - 1) / DT_Y - tile0);
    const int plane0 = sp.slot * v.n_layers;
    auto issue = [&](int kk) {   // one thread: loads of tile kk into stage kk & 1
        constexpr uint32_t kBytes = 3u * DT_R * DT_WT * sizeof(float);
        DetectRaw& r = s.raw[kk & 1];
        uint64_t* bar = &s_bar[kk & 1];
        const int j0 = (tile0 + kk) * DT_Y;
        mbar_expect_tx(bar, kBytes);
        tma_load_3d(&r.P[0][0], &tmap, bar, i0 - DT_HX, j0 - DT_H, plane0 + count_layer);
        tma_load_3d(&r.V[0][0], &tmap, bar, i0 - DT_HX, j0 - DT_H, plane0 + (recompute ? L_M2 : L_VARIANCE));
        tma_load_3d(&r.M[0][0], &tmap, bar, i0 - DT_HX, j0 - DT_H, plane0 + L_MINH);
    };
    if (tid == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
    }
    __syncthreads();
    if (tid == 0) issue(0);
    float* const L0 = v.layer(sp.slot, 0);
    const int i = i0 + tx;
    const int li = tx + DT_HX, lj = ty + DT_H;
    for (int kk = 0; kk < n_tiles; ++kk) {
        // every thread is past the previous tile (barrier at the end of the loop body): its stage may be refilled
        if (tid == 0 && kk + 1 < n_tiles) issue(kk + 1);
        const DetectRaw& raw = s.raw[kk & 1];
        // own cell (overlaps the tile transfer)
        const int j = (tile0 + kk) * DT_Y + ty;
        const bool live = i < N && j < N;
        const int cell = i + j * N;
        float g = 0.0f, c = 0.0f;
        float4 tb = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (live) {
            g = L0[L_GROUND * N2 + cell];
            c = L0[L_GROUNDPATCH * N2 + cell];
            tb = __ldg(sp.detect_tab + cell);
        }
        const int flags = __float_as_int(tb.w);
        mbar_wait(&s_bar[kk & 1], (uint32_t)((kk >> 1) & 1));
        if (recompute) {   // :323 on the tile: V holds m2 (see k_detect_ldg); outside the map 0 / FLT_MIN = 0, as before
            DetectRaw& rw = s.raw[kk & 1];
            for (int p = tid; p < DT_R * DT_WT; p += DT_X * DT_Y) {
                const int row = p / DT_WT, col = p % DT_WT;
                rw.V[row][col] = __fdiv_rn(rw.V[row][col], __fadd_rn(rw.P[row][col], FLT_MIN));
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the stage is refilled by the TMA unit later
            __syncthreads();
            if (live) L0[L_VARIANCE * N2 + cell] = rw.V[lj][li];   // no block reads L_VARIANCE in this mode
        }

        // stage A: column partials of the point counts -- positions p = tid, tid + 256 of the 12 x 40 tile
        // (only columns 0 .. 35 are ever the first row of a window: col + 4 <= 39 stays inside the tile, no bounds tests;
        // together they read every entry of the tile, so they also tell whether all its counts are small integers)
        bool exact = true;
        for (int p = tid; p < DT_R * DT_WC; p += DT_X * DT_Y) {
            const int row = p / DT_WC, col = p % DT_WC;   // row = j index of the tile, col = i index
            float a[5];
#pragma unroll
            for (int q = 0; q < 5; ++q) {
                a[q] = raw.P[row][col + q];
                exact = exact && a[q] >= 0.0f && a[q] <= DT_EXACT_COUNT && a[q] == truncf(a[q]);
            }
            const float c3 = __fadd_rn(__fadd_rn(a[0], a[1]), a[2]);
            s.C3[row][col] = c3;
            s.C5[row][col] = __fadd_rn(__fadd_rn(c3, a[3]), a[4]);
        }
        exact = __syncthreads_and(exact);
        const bool inner = live && (flags & DTF_INNER);
        const bool s5 = (flags & DTF_S5) != 0;
        float psum = 0.0f;
        if (inner && !exact) {   // the window sum in Eigen's order (:359)
            if (s5)
                psum = TreeSum<0, 25>::run([&](int q) { return raw.P[lj - 2 + q / 5][li - 2 + q % 5]; });
            else
                psum = TreeSum<0, 9>::run([&](int q) { return raw.P[lj - 1 + q / 3][li - 1 + q % 3]; });
        } else if (inner) {
            if (s5) {
                const int r0 = li - 2, c0 = lj - 2;
                psum = __fadd_rn(__fadd_rn(__fadd_rn(s.C5[c0][r0], s.C5[c0 + 1][r0]), __fadd_rn(s.C5[c0 + 2][r0], s.C5[c0 + 3][r0])), s.C5[c0 + 4][r0]);
            } else {
                const int r0 = li - 1, c0 = lj - 1;
                psum = __fadd_rn(__fadd_rn(s.C3[c0][r0], s.C3[c0 + 1][r0]), s.C3[c0 + 2][r0]);
            }
        }
        // early skipping of (almost) empty areas, :364 (need is rounded up to float: the float compare is the double one)
        const bool cand = inner && !(psum < tb.x);
        const bool any = __syncthreads_or(cand);
        bool changed = false;
        if (any) {
            // stage B: products, pairs, triples and column minima
            // (products are needed up to column 37 -- the last row of the right-most window --, pairs up to 36, the rest up
            // to 35; reads of columns 40 / 41 for those two extra columns stay inside this struct and feed unused entries)
            for (int p = tid; p < DT_R * DT_WB; p += DT_X * DT_Y) {
                const int row = p / DT_WB, col = p % DT_WB;
                float qv[3], qm[3], m[5];
#pragma unroll
                for (int q = 0; q < 5; ++q) m[q] = raw.M[row][col + q];
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const float pp = raw.P[row][col + q];
                    const float vv = raw.V[row][col + q];
                    qv[q] = __fmul_rn(pp, vv);
                    qm[q] = __fmul_rn(pp, m[q]);
                }
                s.QV[row][col] = qv[0];
                s.QM[row][col] = qm[0];
                const float pv12 = __fadd_rn(qv[1], qv[2]), pm12 = __fadd_rn(qm[1], qm[2]);
                s.PV2[row][col] = __fadd_rn(qv[0], qv[1]);
                s.PM2[row][col] = __fadd_rn(qm[0], qm[1]);
                s.TV[row][col] = __fadd_rn(qv[0], pv12);
                s.TM[row][col] = __fadd_rn(qm[0], pm12);
                const float n3 = min_skip_nan(min_skip_nan(m[0], m[1]), m[2]);
                s.N3[row][col] = n3;
                s.N5[row][col] = min_skip_nan(min_skip_nan(n3, m[3]), m[4]);
            }
            __syncthreads();
            if (cand) {
                const float variance = raw.V[lj][li], centerP = raw.P[lj][li];
                if (s5) {
                    const int r0 = li - 2, c0 = lj - 2;
                    float localmin = s.N5[c0][r0];
#pragma unroll
                    for (int q = 1; q < 5; ++q) {
                        const float t = s.N5[c0 + q][r0];
                        localmin = (t < localmin) ? t : localmin;
                    }
                    const float m0 = raw.M[c0][r0];
                    localmin = (m0 != m0) ? m0 : localmin;
                    changed = detect_decide<5>(kc, psum, localmin, tree25(s.QV, s.PV2, s.TV, r0, c0), tree25(s.QM, s.PM2, s.TM, r0, c0), centerP, variance,
                                               tb.y, tb.z, g, c);
                } else {
                    const int r0 = li - 1, c0 = lj - 1;
                    float localmin = s.N3[c0][r0];
#pragma unroll
                    for (int q = 1; q < 3; ++q) {
                        const float t = s.N3[c0 + q][r0];
                        localmin = (t < localmin) ? t : localmin;
                    }
                    const float m0 = raw.M[c0][r0];
                    localmin = (m0 != m0) ? m0 : localmin;
                    changed = detect_decide<3>(kc, psum, localmin, tree9s(s.QV, s.PV2, r0, c0), tree9s(s.QM, s.PM2, r0, c0), centerP, variance, tb.y, tb.z, g, c);
                }
            }
        }
        if (live) {
            if (changed) {
                L0[L_GROUND * N2 + cell] = g;
                L0[L_GROUNDPATCH * N2 + cell] = c;
            }
            if (v.skew.sk) {
                skew_store_cell(v, sp, cell, i, j, g, c, (flags & DTF_FAR) != 0);
            } else if (v.spiral_recs) {
                const float d1 = decay_confidence(kc, c);
                float* D1 = v.roll_scratch + (size_t)sp.slot * 2 * k.N2;
                D1[cell] = d1;
                if (i == j) D1[k.N2 + cell] = decay_confidence(kc, d1);
            }
        }
        __syncthreads();   // the derived arrays and this stage are free again
    }
}

int launch_build_detect_table(const View& v, const CfgConst& c, float4* tab, cudaStream_t st) {
    k_build_detect_table<<<(v.k.N2 + 255) / 256, 256, 0, st>>>(v, c, tab);
    return 1;
}

// ------------------------------------------------------------------------------------------
// phase 3: spiral interpolation as a level-scheduled wavefront (one CTA per scan).
// The schedule (host-built from the exact RAW/WAR/WAW dependency DAG of the sequential
// sweep, GroundSegmentation.cpp:413-440) guarantees that visits of one level touch disjoint
// data, so executing levels in order reproduces the sequential result bit for bit.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SPIRAL_THREADS) k_spiral(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.x];
    const Const& k = v.k;
    const CfgConst& kc = sp.cfg;
    const int N = k.N;
    float* G = v.layer(sp.slot, L_GROUND);
    float* C = v.layer(sp.slot, L_GROUNDPATCH);
    const int cidx = N / 2 - 1;
    if (threadIdx.x == 0) {
        C[cidx + cidx * N] = 1.0f;          // :405
        G[cidx + cidx * N] = sp.base_z_f;   // :411
    }
    __syncthreads();
    const float fc = (float)cidx;
    for (int lvl = 0; lvl < v.levels; ++lvl) {
        const int b = v.level_start[lvl], e = v.level_start[lvl + 1];
        for (int t = b + threadIdx.x; t < e; t += SPIRAL_THREADS) {
            const uint32_t vis = v.visits[t];
            const int x = (int)(vis & 0xffffu), y = (int)(vis >> 16);
            float cc[9], pr[9];
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                const int g = (x - 1 + q % 3) + (y - 1 + q / 3) * N;
                cc[q] = C[g];
                pr[q] = __fmul_rn(cc[q], G[g]);
            }
            const float h = G[x + y * N];
            const float occ = cc[4];
            const float s = __fadd_rn(tree9(cc), FLT_MIN);  // :457
            const float avg = __fdiv_rn(tree9(pr), s);      // :458
            G[x + y * N] = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, occ), avg), __fmul_rn(occ, h));  // :460
            const float fx = __fsub_rn((float)x, fc), fy = __fsub_rn((float)y, fc);
            const double d2 = __dmul_rn(__dadd_rn(__dmul_rn((double)fx, (double)fx), __dmul_rn((double)fy, (double)fy)), k.res_sq);
            if (d2 > 12.0) {  // :463
                const double o = (double)occ;
                const double dec = __dsub_rn(o, __ddiv_rn(o, kc.dec_factor));
                C[x + y * N] = (float)((dec < 0.001) ? 0.001 : dec);  // std::max(dec, 0.001)
            }
        }
        __syncthreads();
    }
}

// Pipelined wavefront.  Same schedule, same arithmetic, but the per-level critical path no
// longer contains a global-memory round trip:
//   * schedule records are fetched DIST+1 levels ahead, the 3x3 neighbourhoods of G and C (and
//     the pre-decayed confidence) DIST levels ahead, so their L2 latency overlaps earlier levels;
//   * values written fewer than DIST levels before a visit cannot come from that prefetch; the
//     record names them (neighbour index + producer slot) and they travel through a small
//     shared-memory ring written by every visit;
//   * the fp64 confidence decay is read from the table k_detect prepared.
// Per level: barrier -> <= 3 shared loads -> 9 mul, tree sum, div, 2 mul + add -> stores.
template <int THREADS, int DIST>
__global__ void __launch_bounds__(THREADS) k_spiral_pipe(View v, const SlotParams* __restrict__ batch) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    int* s_ls = reinterpret_cast<int*>(s_raw);
    const int L = v.levels;
    float2* xch = reinterpret_cast<float2*>(s_raw + (size_t)((L + 4) & ~3) * sizeof(int));  // [DIST + 1][THREADS]
    const SlotParams& sp = batch[blockIdx.x];
    const Const& k = v.k;
    const int N = k.N;
    const int tid = threadIdx.x;
    float* G = v.layer(sp.slot, L_GROUND);
    float* C = v.layer(sp.slot, L_GROUNDPATCH);
    const float* D1 = v.roll_scratch + (size_t)sp.slot * 2 * k.N2;
    const float* D2 = D1 + k.N2;
    const uint4* __restrict__ recs = v.spiral_recs;
    for (int t = tid; t <= L; t += THREADS) s_ls[t] = v.level_start[t];
    const int cidx = N / 2 - 1;
    if (tid == 0) {
        C[cidx + cidx * N] = 1.0f;          // :405
        G[cidx + cidx * N] = sp.base_z_f;   // :411
    }
    __syncthreads();

    // pipeline state: rec[s] / act[s] describe this thread's visit at level lvl + s
    uint4 rec[DIST + 1];
    bool act[DIST + 1];
    float cc[DIST][9], gg[DIST][9], dd[DIST];
#pragma unroll
    for (int s = 0; s <= DIST; ++s) {
        act[s] = (s < L) && (tid < s_ls[s + 1] - s_ls[s]);
        rec[s] = act[s] ? recs[s_ls[s] + tid] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int s = 0; s < DIST; ++s) {
        dd[s] = 0.0f;
#pragma unroll
        for (int q = 0; q < 9; ++q) cc[s][q] = gg[s][q] = 0.0f;
        if (act[s]) {
            const int x = (int)(rec[s].x & 0xffffu), y = (int)(rec[s].x >> 16);
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                const int g = (x - 1 + q % 3) + (y - 1 + q / 3) * N;
                cc[s][q] = C[g];
                gg[s][q] = G[g];
            }
            dd[s] = (rec[s].w & 2u) ? D2[x + y * N] : D1[x + y * N];
        }
    }

    int buf = 0;  // lvl % (DIST + 1)
    for (int lvl = 0; lvl < L; ++lvl) {
        // (1) prefetch: neighbourhood of the visit at lvl + DIST, record of lvl + DIST + 1
        float ncc[9], ngg[9], ndd = 0.0f;
#pragma unroll
        for (int q = 0; q < 9; ++q) ncc[q] = ngg[q] = 0.0f;
        if (act[DIST]) {
            const int x = (int)(rec[DIST].x & 0xffffu), y = (int)(rec[DIST].x >> 16);
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                const int g = (x - 1 + q % 3) + (y - 1 + q / 3) * N;
                ncc[q] = C[g];
                ngg[q] = G[g];
            }
            ndd = (rec[DIST].w & 2u) ? D2[x + y * N] : D1[x + y * N];
        }
        uint4 nrec = make_uint4(0, 0, 0, 0);
        bool nact = false;
        {
            const int l2 = lvl + DIST + 1;
            if (l2 < L) {
                nact = tid < s_ls[l2 + 1] - s_ls[l2];
                if (nact) nrec = recs[s_ls[l2] + tid];
            }
        }
        // (2) this level's visit
        if (act[0]) {
            const uint32_t ents[4] = {rec[0].y & 0xffffu, rec[0].y >> 16, rec[0].z & 0xffffu, rec[0].z >> 16};
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const uint32_t e = ents[r];
                const int back = (int)(e >> 14);  // written `back` levels ago (0: unused entry)
                if (back) {
                    int b = buf - back;
                    if (b < 0) b += DIST + 1;
                    const float2 val = xch[b * THREADS + (int)(e & 1023u)];
                    const int q = (int)((e >> 10) & 15u);
#pragma unroll
                    for (int qq = 0; qq < 9; ++qq)
                        if (q == qq) {
                            gg[0][qq] = val.x;
                            cc[0][qq] = val.y;
                        }
                }
            }
            const int x = (int)(rec[0].x & 0xffffu), y = (int)(rec[0].x >> 16);
            float pr[9];
#pragma unroll
            for (int q = 0; q < 9; ++q) pr[q] = __fmul_rn(cc[0][q], gg[0][q]);
            const float occ = cc[0][4], h = gg[0][4];
            const float ssum = __fadd_rn(tree9(cc[0]), FLT_MIN);  // :457
            const float avg = __fdiv_rn(tree9(pr), ssum);         // :458
            const float newg = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, occ), avg), __fmul_rn(occ, h));  // :460
            const bool far = (rec[0].w & 1u) != 0u;               // :463 (geometry only, evaluated on the host)
            const float newc = far ? dd[0] : occ;                 // :464 (table from k_detect)
            xch[buf * THREADS + tid] = make_float2(newg, newc);
            G[x + y * N] = newg;
            if (far) C[x + y * N] = newc;
        }
        __syncthreads();
        // (3) advance the pipeline by one level
#pragma unroll
        for (int s = 0; s + 1 < DIST; ++s) {
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                cc[s][q] = cc[s + 1][q];
                gg[s][q] = gg[s + 1][q];
            }
            dd[s] = dd[s + 1];
        }
#pragma unroll
        for (int q = 0; q < 9; ++q) {
            cc[DIST - 1][q] = ncc[q];
            gg[DIST - 1][q] = ngg[q];
        }
        dd[DIST - 1] = ndd;
#pragma unroll
        for (int s = 0; s < DIST; ++s) {
            rec[s] = rec[s + 1];
            act[s] = act[s + 1];
        }
        rec[DIST] = nrec;
        act[DIST] = nact;
        buf = (buf + 1 == DIST + 1) ? 0 : buf + 1;
    }
}

// ------------------------------------------------------------------------------------------
// Skewed-layout spiral.  k_detect copies G, C (and the confidence each visit will store) into
// (side, level, ring) order (skew_store_cell), k_spiral_skew runs the wavefront there with
// coalesced accesses and also stores every result to the normal layers.  See
// gg_host.cpp:build_spiral_skew for the layout.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 spiral_visit(const float2* nb, float d) {
    float cc[9], pr[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) {
        cc[q] = nb[q].y;
        pr[q] = __fmul_rn(nb[q].y, nb[q].x);
    }
    const float occ = cc[4], h = nb[4].x;
    const float ssum = __fadd_rn(tree9(cc), FLT_MIN);  // :457
    const float avg = __fdiv_rn(tree9(pr), ssum);      // :458
    const float newg = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, occ), avg), __fmul_rn(occ, h));  // :460
    return make_float2(newg, skew_decays(d) ? d : occ);  // :463-464 via the table of k_skew
}

// The level time of this kernel is set by the longest per-warp INSTRUCTION sequence between two
// barriers (one SM, a handful of active warps: a warp issues its dependent instructions a few
// cycles apart), not by memory.  So both roles keep their per-level code short: lane threads are
// compiled per side (compile-time neighbour index of the lane's previous cell, running pointers),
// and the irregular visits are spread over 64 threads (one thread per (visit, neighbour) gathers,
// one thread per visit computes; SKEW_IRR_THREADS in all) instead of unrolled in one thread.
constexpr int SKEW_RING = 16;      // levels of irregular-visit blocks kept in shared memory
constexpr int SKEW_STAGE_LEAD = 10;  // a block is staged this many levels before its visits run

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

template <int SIDE>
__device__ __forceinline__ void skew_lane_thread(const View& v, const SlotParams& sp, float2* s_xch) {
    const SkewView& w = v.skew;
    constexpr int XM = SKEW_XCH_DEPTH - 1;   // exchange ring: entry of level l is [l & XM]
    constexpr int PQ = SIDE == 0 ? 1 : (SIDE == 1 ? 3 : (SIDE == 2 ? 7 : 5));  // neighbour index of the lane's previous cell
    constexpr int PF_FAR = 8, PF_NEAR = 2;
    const int L = w.levels, KP = w.KP, lanes = w.lanes, M = w.M;
    const int m = threadIdx.x - SIDE * M;  // this thread walks rings m - 1, m - 1 + M, m - 1 + 2M, ... of side SIDE
    float2* __restrict__ SK = w.sk + (size_t)sp.slot * w.slots;
    const float* __restrict__ SD = w.sd + (size_t)sp.slot * w.slots;
    float* __restrict__ Gn = v.layer(sp.slot, L_GROUND);
    float* __restrict__ Cn = v.layer(sp.slot, L_GROUNDPATCH);
    const int cstep = SIDE == 0 ? v.k.N : (SIDE == 1 ? 1 : (SIDE == 2 ? -v.k.N : -1));  // the lane walks +y, +x, -y, -x
    int off[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) off[q] = w.pattern[SIDE * 9 + q];
    // The only slot a regular visit touches for the first time (i.e. that still sits in HBM / L2) is
    // the newest row of its outer ring, plus its SD entry; everything else was read by this SM a
    // few levels ago.  Those two are prefetched PF_FAR levels ahead into L2 and PF_NEAR levels ahead
    // into L1, so the one-level-ahead loads below are cache hits.
    int off_new = off[0];
#pragma unroll
    for (int q = 1; q < 9; ++q) off_new = max(off_new, off[q]);

    // current phase: level range [lb, le) of the regular run, slot of level l = base0 + l * KP,
    // cell of level l = cell0 + l * cstep, exchange-buffer index xid
    int ph = -1, lb = 0, le = 0, base0 = 0, cell0 = 0, xid = 0;
    int w_first = 0, w_last = 0;  // levels in which any lane of this warp has work (or prefetches)
    auto next_phase = [&]() {
        ++ph;
        const size_t e = ((size_t)ph * 4 + SIDE) * M + m;
        const int col = ph * M + m;
        lb = w.ph_begin[e];
        le = w.ph_end[e];
        base0 = (SIDE * w.rows + w.row0) * KP + col;
        cell0 = w.ph_cell0[e] - lb * cstep;
        xid = SIDE * KP + col;
    };
    auto warp_window = [&]() {
        w_first = lb < le ? lb - PF_FAR : 0x7fffffff;
        w_last = lb < le ? le : -1;
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            w_first = min(w_first, __shfl_xor_sync(0xffffffffu, w_first, d));
            w_last = max(w_last, __shfl_xor_sync(0xffffffffu, w_last, d));
        }
        w_first = max(w_first, 0) & ~1;  // iterations cover two levels
    };
    next_phase();
    warp_window();

    float2 A[9], B[9];
    float dA = -1.0f, dB = -1.0f;
#pragma unroll
    for (int q = 0; q < 9; ++q) A[q] = B[q] = make_float2(0.f, 0.f);
    if (lb == 0 && le > 0) {
#pragma unroll
        for (int q = 0; q < 9; ++q) A[q] = SK[base0 + off[q]];
        dA = SD[base0];
    }
    // two levels per iteration, alternating register sets (a copy would wait for the loads)
#define GG_LANE_LEVEL(l_, CUR, CURD, NXT, NXTD)                                                      \
    {                                                                                               \
        const int l__ = (l_);                                                                       \
        if (l__ + PF_FAR >= lb && l__ + PF_FAR < le) {                                              \
            prefetch_l2(SK + (base0 + (l__ + PF_FAR) * KP + off_new));                              \
            prefetch_l2(SD + (base0 + (l__ + PF_FAR) * KP));                                        \
        }                                                                                           \
        if (l__ + PF_NEAR >= lb && l__ + PF_NEAR < le) {                                            \
            prefetch_l1(SK + (base0 + (l__ + PF_NEAR) * KP + off_new));                             \
            prefetch_l1(SD + (base0 + (l__ + PF_NEAR) * KP));                                       \
        }                                                                                           \
        if (l__ + 1 >= lb && l__ + 1 < le) {                                                        \
            const float2* p__ = SK + (base0 + (l__ + 1) * KP);                                      \
            _Pragma("unroll") for (int q = 0; q < 9; ++q) NXT[q] = p__[off[q]];                    \
            NXTD = SD[base0 + (l__ + 1) * KP];                                                      \
        }                                                                                           \
        if (l__ >= lb && l__ < le) {                                                                \
            CUR[PQ] = s_xch[((l__ - 1) & XM) * lanes + xid];                                        \
            const float2 r__ = spiral_visit(CUR, CURD);                                             \
            s_xch[(l__ & XM) * lanes + xid] = r__;                                                  \
            SK[base0 + l__ * KP] = r__;                                                             \
            Gn[cell0 + l__ * cstep] = r__.x;                                                        \
            if (skew_decays(CURD)) Cn[cell0 + l__ * cstep] = r__.y;                                 \
        }                                                                                           \
        __syncthreads();                                                                            \
    }
    for (int l = 0; l < L; l += 2) {
        // done with this ring: move on to ring + M (it starts well after this one ended)
        if (w.phases > 1) {
            bool moved = false;
            while (ph + 1 < w.phases && l >= le) {
                next_phase();
                moved = true;
            }
            if (__any_sync(0xffffffffu, moved)) warp_window();
        }
        // a warp (32 consecutive rings of one side) has work only in a window of levels; outside of it
        // the per-level cost must be the barrier alone (the level time is set by instruction issue)
        if (l < w_first || l >= w_last) {
            __syncthreads();
            if (l + 1 < L) __syncthreads();
            continue;
        }
        GG_LANE_LEVEL(l, A, dA, B, dB)
        if (l + 1 < L) GG_LANE_LEVEL(l + 1, B, dB, A, dA)
    }
#undef GG_LANE_LEVEL
}

__device__ __forceinline__ void skew_named_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(SKEW_IRR_THREADS) : "memory"); }

__device__ __forceinline__ void skew_irregular_thread(const View& v, const SlotParams& sp, float2* s_xch, uint4* s_ring, float2* s_nb, float* s_dd) {
    const SkewView& w = v.skew;
    const int ti = threadIdx.x - 4 * w.M;  // 0 .. 63
    constexpr int XM = SKEW_XCH_DEPTH - 1;
    const int L = w.levels, lanes = w.lanes;
    const int chunks = w.irr_chunks, irr_max = w.irr_max;
    float2* __restrict__ SK = w.sk + (size_t)sp.slot * w.slots;
    const float* __restrict__ SD = w.sd + (size_t)sp.slot * w.slots;
    const uint4* __restrict__ blocks = w.irr_blocks;
    float* __restrict__ Gn = v.layer(sp.slot, L_GROUND);
    float* __restrict__ Cn = v.layer(sp.slot, L_GROUNDPATCH);
    if (ti == 0) {  // spiral_ground_interpolation :405,411 on the normal layers (the skewed copy has it from k_detect)
        const int cidx = v.k.N / 2 - 1;
        Cn[cidx + cidx * v.k.N] = 1.0f;
        Gn[cidx + cidx * v.k.N] = sp.base_z_f;
    }
    const uint32_t* ring_w = reinterpret_cast<const uint32_t*>(s_ring);
    const int ring_words = chunks * 4;
    const bool stager = ti < chunks;              // copies one 16-byte chunk of the level blocks per level
    const bool gatherer = ti < irr_max * 9;       // (visit ti / 9, neighbour ti % 9)
    const bool visitor = ti < irr_max;            // computes visit ti

    // prologue: blocks of levels 0 .. LEAD-1 -> ring; gather of level 0; block of level LEAD in flight
    if (stager) {
        for (int b = 0; b < SKEW_STAGE_LEAD; ++b) s_ring[b * chunks + ti] = blocks[(size_t)min(b, L + 3) * chunks + ti];  // the table has 4 padding levels
    }
    uint4 stage = stager ? blocks[(size_t)min(SKEW_STAGE_LEAD, L + 3) * chunks + ti] : make_uint4(0, 0, 0, 0);
    skew_named_barrier();
    float2 val = make_float2(0.f, 0.f);
    float dval = -1.0f;
    uint32_t info = 0xffffffffu;
    bool have = false;
    if (gatherer) {
        const uint32_t slot = ring_w[0 * ring_words + ti * 2], rl = ring_w[0 * ring_words + ti * 2 + 1];
        have = slot != 0xffffffffu;
        if (have) {
            val = SK[slot];
            info = rl;
            if (ti % 9 == 4) dval = SD[slot];
        }
    }
    for (int l = 0; l < L; ++l) {
        // (1) block of level l + LEAD (loaded during the previous level) -> ring; start loading the next one
        if (stager) {
            s_ring[((l + SKEW_STAGE_LEAD) % SKEW_RING) * chunks + ti] = stage;
            stage = blocks[(size_t)min(l + SKEW_STAGE_LEAD + 1, L + 3) * chunks + ti];
        }
        // (2) hand the gathered neighbour of THIS level to the visitor, gather the one of level l + 1,
        //     pull the one of level l + LEAD - 2 towards L2 / L1
        if (gatherer) {
            if (have) {
                if (info != 0xffffffffu) val = s_xch[((l - 1) & XM) * lanes + (int)info];  // written at level l - 1
                s_nb[ti] = val;
                if (ti % 9 == 4) s_dd[ti / 9] = dval;
            }
            const uint32_t far_slot = ring_w[((l + SKEW_STAGE_LEAD - 2) % SKEW_RING) * ring_words + ti * 2];
            if (far_slot != 0xffffffffu) {
                prefetch_l2(SK + far_slot);
                if (ti % 9 == 4) prefetch_l2(SD + far_slot);
            }
            const uint32_t near_slot = ring_w[((l + 3) % SKEW_RING) * ring_words + ti * 2];
            if (near_slot != 0xffffffffu) {
                prefetch_l1(SK + near_slot);
                if (ti % 9 == 4) prefetch_l1(SD + near_slot);
            }
            const uint32_t* e = ring_w + ((l + 1) % SKEW_RING) * ring_words + ti * 2;
            const uint32_t slot = e[0];
            have = (l + 1 < L) && slot != 0xffffffffu;
            if (have) {
                val = SK[slot];
                info = e[1];
                if (ti % 9 == 4) dval = SD[slot];
            }
        }
        skew_named_barrier();
        // (3) the visits of this level
        if (visitor) {
            const uint32_t* hd = ring_w + (l % SKEW_RING) * ring_words + irr_max * 18 + ti * 4;
            const uint32_t own = hd[0];
            if (own != 0xffffffffu) {
                float2 nb[9];
#pragma unroll
                for (int q = 0; q < 9; ++q) nb[q] = s_nb[ti * 9 + q];
                const float2 r = spiral_visit(nb, s_dd[ti]);
                const int mirror = (int)hd[1];
                s_xch[(l & XM) * lanes + (int)hd[2]] = r;
                SK[own] = r;
                if (mirror >= 0) SK[mirror] = r;
                Gn[hd[3]] = r.x;
                if (skew_decays(s_dd[ti])) Cn[hd[3]] = r.y;
            }
        }
        __syncthreads();
    }
}

template <int MAXT, int MIN_CTAS = 1>
__global__ void __launch_bounds__(MAXT, MIN_CTAS) k_spiral_skew(View v, const SlotParams* __restrict__ batch) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    const SkewView& w = v.skew;
    // [ring: SKEW_RING levels x irr_chunks uint4][xch: SKEW_XCH_DEPTH x lanes float2][nb: irr_max*9 float2][dd: irr_max float]
    uint4* s_ring = reinterpret_cast<uint4*>(s_raw);
    float2* s_xch = reinterpret_cast<float2*>(s_ring + SKEW_RING * w.irr_chunks);
    float2* s_nb = s_xch + SKEW_XCH_DEPTH * w.lanes;
    float* s_dd = reinterpret_cast<float*>(s_nb + w.irr_max * 9);
    const SlotParams& sp = batch[blockIdx.x];
    const int tid = threadIdx.x;
    if (tid < 4 * w.M) {
        const int side = tid / w.M;  // warp-uniform: M is a multiple of 32
        if (side == 0)
            skew_lane_thread<0>(v, sp, s_xch);
        else if (side == 1)
            skew_lane_thread<1>(v, sp, s_xch);
        else if (side == 2)
            skew_lane_thread<2>(v, sp, s_xch);
        else
            skew_lane_thread<3>(v, sp, s_xch);
    } else {
        skew_irregular_thread(v, sp, s_xch, s_ring, s_nb, s_dd);
    }
}

// ------------------------------------------------------------------------------------------
// phase 4: labelling (:146-196)
// ------------------------------------------------------------------------------------------
// LABEL_ILP points per thread (strided by the block, so every access stays coalesced): the streaming loads of all
// of them are issued first, then the two gathers each, then the arithmetic -- the kernel is bound by memory latency.
constexpr int LABEL_ILP = 4;

__global__ void __launch_bounds__(256) k_label(View v, const SlotParams* __restrict__ batch) {
    const SlotParams& sp = batch[blockIdx.y];
    const Const& k = v.k;
    const size_t base = (size_t)sp.slot * v.pcap;
    const int i0 = blockIdx.x * (256 * LABEL_ILP) + threadIdx.x;
    const int n = sp.n_points;
    if (i0 >= n) return;
    const float* L0 = v.layer(sp.slot, 0);
    const float* G = L0 + L_GROUND * k.N2;
    const float* V = L0 + L_VARIANCE * k.N2;
    float* OBS = v.layer(sp.slot, L_OBSTACLES);

    uint32_t code[LABEL_ILP];
    float dist[LABEL_ILP], z[LABEL_ILP], gh[LABEL_ILP], var[LABEL_ILP];
#pragma unroll
    for (int u = 0; u < LABEL_ILP; ++u) {
        const int i = i0 + u * 256;
        const bool in = i < n;
        code[u] = in ? v.code[base + i] : (PC_ABSENT << 24);
        dist[u] = in ? v.dist[base + i] : 0.0f;
        z[u] = in ? __uint_as_float(v.zw[base + i].x) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < LABEL_ILP; ++u) {
        const uint32_t cls = code[u] >> 24;
        const int cell = (int)(code[u] & 0xffffffu);
        const bool use = cls == PC_KEPT || cls == PC_IGNORED;
        gh[u] = use ? G[cell] : 0.0f;
        var[u] = use ? V[cell] : 1.0f;
    }
#pragma unroll
    for (int u = 0; u < LABEL_ILP; ++u) {
        const int i = i0 + u * 256;
        if (i >= n) break;
        const uint32_t cls = code[u] >> 24;
        const int cell = (int)(code[u] & 0xffffffu);
        uint8_t label = GG_LABEL_ABSENT;
        if (cls == PC_OUTLIER) {
            label = GG_LABEL_GROUND;
        } else if (cls == PC_KEPT || cls == PC_IGNORED) {
            const double groundheight = (double)gh[u];
            // std::max(std::min((f * dist) / variance * thres, thres), obs_thres) with C++ min/max semantics
            const double lab_fac = sp.cfg.lab_fac, lab_thres = sp.cfg.lab_thres, lab_obs = sp.cfg.lab_obs;
            const double a = __dmul_rn(__ddiv_rn(__dmul_rn(lab_fac, (double)dist[u]), (double)var[u]), lab_thres);
            double t = (lab_thres < a) ? lab_thres : a;
            t = (t < lab_obs) ? lab_obs : t;
            if (__dadd_rn(t, groundheight) < (double)z[u]) {
                label = GG_LABEL_NONGROUND;
                atomicAdd(OBS + cell, 1.0f);  // small exact integers: order free
            } else {
                label = GG_LABEL_GROUND;
            }
        }
        v.labels[base + i] = label;
    }
}

// ------------------------------------------------------------------------------------------
// output cloud order: kept (input order), ignored (input order), outliers (input order)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int out_class(uint32_t code) {
    const uint32_t cls = code >> 24;
    return cls == PC_KEPT ? 0 : (cls == PC_IGNORED ? 1 : (cls == PC_OUTLIER ? 2 : -1));
}

// out_class of input point i of a scan, or -1 when its label is not in `select` (GG_SELECT_*; outliers are ground)
__device__ __forceinline__ int out_class_selected(const View& v, size_t base, int i, int n, unsigned select) {
    if (i >= n) return -1;
    const int c = out_class(v.code[base + i]);
    if (c < 0 || select == (GG_SELECT_GROUND | GG_SELECT_NONGROUND)) return c;
    const unsigned bit = (v.labels[base + i] == GG_LABEL_NONGROUND) ? GG_SELECT_NONGROUND : GG_SELECT_GROUND;
    return (select & bit) ? c : -1;
}

__global__ void __launch_bounds__(OUT_TILE) k_out_count(View v, const SlotParams* __restrict__ batch, const OutDest* __restrict__ dests,
                                                        int nblk) {
    const SlotParams& sp = batch[blockIdx.y];
    const int i = blockIdx.x * OUT_TILE + threadIdx.x;
    const int c = out_class_selected(v, (size_t)sp.slot * v.pcap, i, sp.n_points, dests[blockIdx.y].select);
    int* counts = v.out_counts + (size_t)sp.slot * (3 * v.out_blocks + 1);
    const int n0 = __syncthreads_count(c == 0);
    const int n1 = __syncthreads_count(c == 1);
    const int n2 = __syncthreads_count(c == 2);
    if (threadIdx.x == 0) {
        counts[0 * nblk + blockIdx.x] = n0;
        counts[1 * nblk + blockIdx.x] = n1;
        counts[2 * nblk + blockIdx.x] = n2;
    }
}

__global__ void __launch_bounds__(1024) k_out_scan(View v, const SlotParams* __restrict__ batch, const OutDest* __restrict__ dests, int nblk) {
    const SlotParams& sp = batch[blockIdx.x];
    int* counts = v.out_counts + (size_t)sp.slot * (3 * v.out_blocks + 1);
    const int total = block_exclusive_scan_1024(counts, counts, 3 * nblk);
    if (threadIdx.x == 0) {
        counts[3 * v.out_blocks] = total;
        if (int* dc = dests[blockIdx.x].count) *dc = total;
    }
}

__global__ void __launch_bounds__(OUT_TILE) k_out_write(View v, const SlotParams* __restrict__ batch, const OutDest* __restrict__ dests,
                                                        int nblk) {
    __shared__ int s_w[3][32];
    const SlotParams& sp = batch[blockIdx.y];
    const OutDest d = dests[blockIdx.y];
    const size_t base = (size_t)sp.slot * v.pcap;
    const int i = blockIdx.x * OUT_TILE + threadIdx.x;
    if (d.labels && i < sp.n_points) d.labels[i] = v.labels[base + i];
    if (!d.index && !d.cloud) return;  // the same for the whole block
    const int c = out_class_selected(v, base, i, sp.n_points, d.select);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    int rank_in_warp = 0;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const uint32_t bal = __ballot_sync(0xffffffffu, c == q);
        if (c == q) rank_in_warp = __popc(bal & lt_mask);
        if (lane == 0) s_w[q][warp] = __popc(bal);
    }
    __syncthreads();
    if (warp < 3) {  // warp q scans the 32 warp totals of class q
        const int w = s_w[warp][lane];
        const int wi = warp_inclusive_scan(w);
        s_w[warp][lane] = wi - w;
    }
    __syncthreads();
    if (c < 0) return;
    const int* counts = v.out_counts + (size_t)sp.slot * (3 * v.out_blocks + 1);
    const int pos = counts[c * nblk + blockIdx.x] + s_w[c][warp] + rank_in_warp;
    if (d.index) d.index[pos] = (uint32_t)i;
    if (d.cloud) {
        const uint4* rec = reinterpret_cast<const uint4*>(sp.src + i);
        uint4 a = rec[0], b = rec[1];
        b.x = __float_as_uint((float)v.labels[base + i]);  // intensity = 49 / 99 (:175,180,188)
        uint4* dst = reinterpret_cast<uint4*>(d.cloud + pos);
        dst[0] = a;
        dst[1] = b;
    }
}

// ------------------------------------------------------------------------------------------
// Batched layer transfer (gg_get_layers_to_device / gg_set_layers_from_device): block (x, s, l) copies LC_ILP * 256
// cells of plane l of scan s between the arena (View::layer) and the caller's buffer, coalesced over the cells.
// N2 may be odd, so the copy stays scalar (4-byte aligned buffers).
// ------------------------------------------------------------------------------------------
constexpr int LC_THREADS = 256;
constexpr int LC_ILP = 4;

template <bool IMPORT>
__global__ void __launch_bounds__(LC_THREADS) k_layer_copy(View v, const SlotParams* __restrict__ batch, LayerList names, float* __restrict__ buf) {
    const SlotParams& sp = batch[blockIdx.y];
    const int l = blockIdx.z;
    const int idx = names.idx[l];
    float* lay = v.layer(sp.slot, idx == LAYER_POINTS ? sp.points_layer : idx);
    float* ext = buf + ((size_t)sp.pos * names.n + l) * v.k.N2;
    const float* __restrict__ src = IMPORT ? ext : lay;
    float* __restrict__ dst = IMPORT ? lay : ext;
    const int i0 = blockIdx.x * (LC_THREADS * LC_ILP) + threadIdx.x;
    float r[LC_ILP];
#pragma unroll
    for (int q = 0; q < LC_ILP; ++q) {
        const int i = i0 + q * LC_THREADS;
        if (i < v.k.N2) r[q] = src[i];
    }
#pragma unroll
    for (int q = 0; q < LC_ILP; ++q) {
        const int i = i0 + q * LC_THREADS;
        if (i < v.k.N2) dst[i] = r[q];
    }
}

// ------------------------------------------------------------------------------------------
// "next" rows (SURVEY.md section 8f)
// ------------------------------------------------------------------------------------------
// f1: pcl::fromROSMsg (field-offset driven unpack, GroundGridNodelet.cpp:119-120) + the per-point
// tf2::doTransform into the map frame in fp64, stored as float (:166-181).  Block (x, s) unpacks 256 points of payload s
// into its slot's cloud buffer, from record descs[s].first on.  The loads are byte-wise: payloads may be unaligned and
// fields sit at any offset (the KITTI player's 18-byte points).
__global__ void __launch_bounds__(256) k_unpack_transform(View v, const SlotParams* __restrict__ batch, const UnpackDesc* __restrict__ descs) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    const SlotParams& sp = batch[blockIdx.y];
    if (i >= sp.n_points) return;
    const UnpackDesc& d = descs[blockIdx.y];
    const unsigned char* p = d.raw + (size_t)i * d.point_step;
    auto rd32 = [&](int off) -> uint32_t {
        if (off < 0) return 0u;
        return (uint32_t)p[off] | ((uint32_t)p[off + 1] << 8) | ((uint32_t)p[off + 2] << 16) | ((uint32_t)p[off + 3] << 24);
    };
    float x = __uint_as_float(rd32(d.off[0])), y = __uint_as_float(rd32(d.off[1])), z = __uint_as_float(rd32(d.off[2]));
    const uint32_t inten = rd32(d.off[3]);
    const uint32_t ring = d.off[4] < 0 ? 0u : ((uint32_t)p[d.off[4]] | ((uint32_t)p[d.off[4] + 1] << 8));
    if (d.transform) {
        const double dx = (double)x, dy = (double)y, dz = (double)z;
        const double* T = d.T;
        // tf2::Transform * Vector3: row.dot(v) (left to right) + origin
        x = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], dx), __dmul_rn(T[1], dy)), __dmul_rn(T[2], dz)), T[3]);
        y = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], dx), __dmul_rn(T[5], dy)), __dmul_rn(T[6], dz)), T[7]);
        z = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], dx), __dmul_rn(T[9], dy)), __dmul_rn(T[10], dz)), T[11]);
    }
    uint4* dst = reinterpret_cast<uint4*>(v.points + (size_t)sp.slot * v.pcap + d.first + i);
    dst[0] = make_uint4(__float_as_uint(x), __float_as_uint(y), __float_as_uint(z), 0u);
    dst[1] = make_uint4(inten, ring, 0u, 0u);
}

// f3: the images of GroundGridNodelet::publish_grid_map_layer (:234-291) for a batch of scans.  Both are the transpose
// of the column-major layers (cv::Mat row = index(0), col = index(1)): block (t, s[, l]) owns an IMG_TILE x IMG_TILE tile
// of the image, reads it along i (coalesced in the layer), and writes it along j (coalesced in the image) through
// shared memory.  Per scan the staging entry carries batch[s].slot, batch[s].pos = its position k in the call and
// batch[s].points_layer (as launch_layer_copy).
constexpr int IMG_TILE = 32;
constexpr int IMG_ROWS = 8;   // blockDim (IMG_TILE, IMG_ROWS): every thread handles IMG_TILE / IMG_ROWS rows of a tile
constexpr int IR_THREADS = 256;
constexpr int IR_ILP = IMG_RANGE_CELLS / IR_THREADS;
// monotone float -> int mapping: integer order is the order of the floats, with -0 below +0
constexpr int KEY_POS_INF = 0x7f800000;                                  // order_key(+inf)
constexpr int KEY_NEG_INF = (int)(0xff800000u ^ 0x7fffffffu);           // order_key(-inf)
__device__ __forceinline__ int order_key(float f) { const int b = __float_as_int(f); return b >= 0 ? b : (b ^ 0x7fffffff); }
__device__ __forceinline__ float order_unkey(int k) { return __int_as_float(k >= 0 ? k : (k ^ 0x7fffffff)); }
__device__ __forceinline__ bool finite_f(float x) { return fabsf(x) <= FLT_MAX; }

__device__ __forceinline__ const float* __restrict__ image_plane(const View& v, const SlotParams& sp, const LayerList& names, int l) {
    const int idx = names.idx[l];
    return v.layer(sp.slot, idx == LAYER_POINTS ? sp.points_layer : idx);
}

// The 8-bit image grid_map::GridMapCvConverter::toImage<unsigned char, 1>(map, layer, CV_8UC1, img) hands to
// cv::applyColorMap (GroundGridNodelet.cpp:238-245): lower / upper = min / max over the finite cells of the layer, pixel
// (i, j) = (unsigned char)(((value - lower) / (upper - lower)) * 255.f), non-finite cells stay 0.
// Pass 1: block (x, s, l) reduces IMG_RANGE_CELLS cells of plane l of scan s to the ordered keys of their finite
// min / max, stored at partial[(slot * L_NUM + l) * gridDim.x + x] (no finite cell: the keys of +inf / -inf).
__global__ void __launch_bounds__(IR_THREADS) k_layer_range(View v, const SlotParams* __restrict__ batch, LayerList names, int2* __restrict__ partial) {
    __shared__ int2 s_warp[IR_THREADS / 32];
    const SlotParams& sp = batch[blockIdx.y];
    const float* __restrict__ lay = image_plane(v, sp, names, blockIdx.z);
    const int i0 = blockIdx.x * IMG_RANGE_CELLS + threadIdx.x;
    float x[IR_ILP];
#pragma unroll
    for (int q = 0; q < IR_ILP; ++q) {
        const int i = i0 + q * IR_THREADS;
        x[q] = i < v.k.N2 ? lay[i] : NAN;
    }
    int lo = KEY_POS_INF, hi = KEY_NEG_INF;
#pragma unroll
    for (int q = 0; q < IR_ILP; ++q)
        if (finite_f(x[q])) {
            const int kx = order_key(x[q]);
            lo = min(lo, kx);
            hi = max(hi, kx);
        }
    lo = __reduce_min_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = make_int2(lo, hi);
    __syncthreads();
    if (threadIdx.x < 32) {
        const int2 w = threadIdx.x < IR_THREADS / 32 ? s_warp[threadIdx.x] : make_int2(KEY_POS_INF, KEY_NEG_INF);
        lo = __reduce_min_sync(0xffffffffu, w.x);
        hi = __reduce_max_sync(0xffffffffu, w.y);
        if (threadIdx.x == 0) partial[((size_t)sp.slot * L_NUM + blockIdx.z) * gridDim.x + blockIdx.x] = make_int2(lo, hi);
    }
}

// Pass 2: block (t, s, l) reduces the n_part partials of plane l of scan s to (lower, upper) and writes tile t of its
// image to dst[(k * names.n + l) * N2 + i * N + j]; the block of tile 0 also stores the range at range[(k * names.n + l) * 2].
__global__ void __launch_bounds__(IMG_TILE * IMG_ROWS) k_layer_image(View v, const SlotParams* __restrict__ batch, LayerList names,
                                                                   const int2* __restrict__ partial, int n_part, unsigned char* __restrict__ dst,
                                                                   float* __restrict__ range) {
    __shared__ unsigned char tile[IMG_TILE][IMG_TILE + 1];   // [j - j0][i - i0]
    __shared__ float s_range[2];
    const SlotParams& sp = batch[blockIdx.y];
    const int l = blockIdx.z, N = v.k.N, tx = threadIdx.x, ty = threadIdx.y;
    const int tiles = (N + IMG_TILE - 1) / IMG_TILE;
    const int i0 = (blockIdx.x % tiles) * IMG_TILE, j0 = (blockIdx.x / tiles) * IMG_TILE;
    const float* __restrict__ lay = image_plane(v, sp, names, l);
    float x[IMG_TILE / IMG_ROWS];
#pragma unroll
    for (int r = 0; r < IMG_TILE / IMG_ROWS; ++r) {
        const int i = i0 + tx, j = j0 + ty + r * IMG_ROWS;
        x[r] = (i < N && j < N) ? lay[i + (size_t)j * N] : 0.0f;
    }
    if (ty == 0) {
        const int2* __restrict__ p = partial + ((size_t)sp.slot * L_NUM + l) * n_part;
        int lo = KEY_POS_INF, hi = KEY_NEG_INF;
        for (int b = tx; b < n_part; b += 32) {
            const int2 q = p[b];
            lo = min(lo, q.x);
            hi = max(hi, q.y);
        }
        lo = __reduce_min_sync(0xffffffffu, lo);
        hi = __reduce_max_sync(0xffffffffu, hi);
        if (tx == 0) {
            s_range[0] = order_unkey(lo);
            s_range[1] = order_unkey(hi);
            if (range && blockIdx.x == 0) {
                float* out = range + ((size_t)sp.pos * names.n + l) * 2;
                out[0] = s_range[0];
                out[1] = s_range[1];
            }
        }
    }
    __syncthreads();
    const float lower = s_range[0], upper = s_range[1];
#pragma unroll
    for (int r = 0; r < IMG_TILE / IMG_ROWS; ++r) {
        unsigned char px = 0;
        if (finite_f(x[r])) {
            const float t = __fmul_rn(__fdiv_rn(__fsub_rn(x[r], lower), __fsub_rn(upper, lower)), 255.0f);
            px = (t == t) ? (unsigned char)(int)t : 0;   // (Type_) cast: truncation; a constant layer (0 / 0) has no defined image
        }
        tile[ty + r * IMG_ROWS][tx] = px;
    }
    __syncthreads();
    unsigned char* __restrict__ img = dst + ((size_t)sp.pos * names.n + l) * v.k.N2;
#pragma unroll
    for (int r = 0; r < IMG_TILE / IMG_ROWS; ++r) {
        const int i = i0 + ty + r * IMG_ROWS, j = j0 + tx;
        if (i < N && j < N) img[(size_t)i * N + j] = tile[tx][ty + r * IMG_ROWS];
    }
}

// The "terrain" image (:247-270): CV_32FC3, pixel (i, j) = (ground height, 3x3 sum of pointsRaw >= 27 ? 1 : 0, pointsRaw).
// The reference reads the 3x3 block out of bounds on the border cells; here border cells get visited = 0.  Block (t, s)
// stages the tile's ground and its pointsRaw with a one-cell halo, then writes each image row of the tile as
// 3 * IMG_TILE consecutive floats to dst[k][i][j][3].
__global__ void __launch_bounds__(IMG_TILE * IMG_ROWS) k_terrain_image(View v, const SlotParams* __restrict__ batch, float* __restrict__ dst) {
    constexpr int H = IMG_TILE + 2;
    __shared__ float s_raw[H][H + 1];               // [j - j0 + 1][i - i0 + 1]
    __shared__ float s_gnd[IMG_TILE][IMG_TILE + 1];  // [j - j0][i - i0]
    const SlotParams& sp = batch[blockIdx.y];
    const int N = v.k.N, tx = threadIdx.x, ty = threadIdx.y;
    const int tiles = (N + IMG_TILE - 1) / IMG_TILE;
    const int i0 = (blockIdx.x % tiles) * IMG_TILE, j0 = (blockIdx.x / tiles) * IMG_TILE;
    const float* __restrict__ raw = v.layer(sp.slot, L_RAW);
    const float* __restrict__ gnd = v.layer(sp.slot, L_GROUND);
    for (int e = ty * IMG_TILE + tx; e < H * H; e += IMG_TILE * IMG_ROWS) {
        const int ii = e % H, jj = e / H, i = i0 - 1 + ii, j = j0 - 1 + jj;
        s_raw[jj][ii] = (i >= 0 && j >= 0 && i < N && j < N) ? raw[i + (size_t)j * N] : 0.0f;
    }
#pragma unroll
    for (int r = 0; r < IMG_TILE / IMG_ROWS; ++r) {
        const int i = i0 + tx, j = j0 + ty + r * IMG_ROWS;
        s_gnd[ty + r * IMG_ROWS][tx] = (i < N && j < N) ? gnd[i + (size_t)j * N] : 0.0f;
    }
    __syncthreads();
    const int w3 = 3 * min(IMG_TILE, N - j0);   // floats of one image row inside the tile
#pragma unroll
    for (int r = 0; r < IMG_TILE / IMG_ROWS; ++r) {
        const int ii = ty + r * IMG_ROWS, i = i0 + ii;
        if (i >= N) break;
        float* __restrict__ row = dst + ((size_t)sp.pos * v.k.N2 + (size_t)i * N + j0) * 3;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const int f = tx + q * IMG_TILE;
            if (f >= w3) break;
            const int jj = f / 3, c = f - 3 * jj, j = j0 + jj;
            float val;
            if (c == 0) {
                val = s_gnd[jj][ii];
            } else if (c == 2) {
                val = s_raw[jj + 1][ii + 1];
            } else {
                val = 0.0f;
                if (i >= 1 && j >= 1 && i < N - 1 && j < N - 1) {
                    float e[9];
#pragma unroll
                    for (int m = 0; m < 9; ++m) e[m] = s_raw[jj + m / 3][ii + m % 3];   // cell (i - 1 + m % 3, j - 1 + m / 3)
                    val = tree9(e) >= 27.0f ? 1.0f : 0.0f;
                }
            }
            row[f] = val;
        }
    }
}

// f4: the tallies of scripts/eval_groundpoint_classifier.py:95-118 for a batch of segmented clouds: per
// ground-truth label id (carried in `ring`, scripts/kitti_data_publisher.py:122-132) the number of
// points predicted ground (49, bin 2 * id) and non-ground (99, bin 2 * id + 1); absent points and ids
// >= EVAL_LABELS are not counted.  Blocks (x, scan): block x tallies points [x, x + 1) * EVAL_TILE of
// scan batch[scan] in a shared histogram, then adds each non-zero bin into the scan's tally at
// counts + batch[scan].pos * 2 * EVAL_LABELS with one 64-bit atomic.  Most points of a scene fall
// into a few ids (road, building, vegetation): the lanes of a warp that hit one bin add once
// (__match_any_sync, as k_rasterize does for its runs).  Per point: the label byte and the ring
// (uint16 of the packed cloud, else the second 16 bytes of the 32-byte record).
constexpr int EVAL_THREADS = 256, EVAL_ILP = 4, EVAL_ROUNDS = 8;
constexpr int EVAL_TILE = EVAL_THREADS * EVAL_ILP * EVAL_ROUNDS;   // points per block
__global__ void __launch_bounds__(EVAL_THREADS) k_eval_counts(View v, const SlotParams* __restrict__ batch, unsigned long long* __restrict__ counts) {
    const SlotParams& sp = batch[blockIdx.y];
    const int n = sp.n_points, tile0 = blockIdx.x * EVAL_TILE;
    if (tile0 >= n) return;   // the grid covers the largest scan of the batch
    __shared__ unsigned int s_cnt[EVAL_LABELS * 2];
    for (int t = threadIdx.x; t < EVAL_LABELS * 2; t += EVAL_THREADS) s_cnt[t] = 0u;
    __syncthreads();
    const uint8_t* labels = v.labels + (size_t)sp.slot * v.pcap;
    const unsigned short* rings = sp.packed ? reinterpret_cast<const unsigned short*>(sp.packed + 3 * ((n + 7) & ~7)) : nullptr;
    const int end = min(n, tile0 + EVAL_TILE), lane = threadIdx.x & 31;
    constexpr unsigned NO_BIN = 0xffffffffu;
    for (int r0 = tile0; r0 < end; r0 += EVAL_THREADS * EVAL_ILP) {   // uniform over the block: whole warps reach the match
        unsigned bin[EVAL_ILP];
#pragma unroll
        for (int u = 0; u < EVAL_ILP; ++u) {
            const int i = r0 + u * EVAL_THREADS + threadIdx.x;
            bin[u] = NO_BIN;
            if (i < end) {
                const unsigned label = labels[i];
                const unsigned ring = rings ? rings[i] : reinterpret_cast<const uint4*>(sp.src + i)[1].y & 0xffffu;
                if (label != GG_LABEL_ABSENT && ring < EVAL_LABELS) bin[u] = ring * 2 + (label == GG_LABEL_NONGROUND ? 1 : 0);
            }
        }
#pragma unroll
        for (int u = 0; u < EVAL_ILP; ++u) {
            // lanes without a point to count get a private pseudo key (never equal to a bin)
            const unsigned peers = __match_any_sync(0xffffffffu, bin[u] != NO_BIN ? bin[u] : (0x80000000u | (unsigned)lane));
            if (bin[u] != NO_BIN && lane == __ffs(peers) - 1) atomicAdd(&s_cnt[bin[u]], (unsigned)__popc(peers));
        }
    }
    __syncthreads();
    unsigned long long* dst = counts + (size_t)sp.pos * (EVAL_LABELS * 2);
    for (int t = threadIdx.x; t < EVAL_LABELS * 2; t += EVAL_THREADS)
        if (s_cnt[t]) atomicAdd(&dst[t], (unsigned long long)s_cnt[t]);
}

// Terrain lookups (gg_sample_layers_to_device).  Blocks (x, set): every thread takes SAMPLE_ILP queries of set
// batch[set] SAMPLE_THREADS apart, issues their position loads up front (as k_label does), finds each query's cell with
// the rasterizer's grid_index / grid_inside and, in linear mode, its bilinear weights once; then per name it gathers 1
// or 4 cells per query and stores the values coalesced at dst[l * n + q].  Arithmetic: fp64, correctly rounded, no
// contraction (the header's definition).  A linear value that is NaN, and every value outside the map, is stored as
// the quiet NaN 0x7fc00000 (device fp64 arithmetic does not keep NaN payloads); nearest values keep their bits.
constexpr int SAMPLE_THREADS = 256, SAMPLE_ILP = 2;   // 4 queries per thread need 107 registers; 2 keep 64 and four blocks per SM
constexpr uint32_t SAMPLE_NAN = 0x7fc00000u;

__global__ void __launch_bounds__(SAMPLE_THREADS) k_sample_layers(View v, const SlotParams* __restrict__ batch, const QueryDesc* __restrict__ descs,
                                                                  LayerList names, int mode) {
    const SlotParams& sp = batch[blockIdx.y];
    const unsigned n = (unsigned)sp.n_points;
    const unsigned q0 = blockIdx.x * (SAMPLE_THREADS * SAMPLE_ILP) + threadIdx.x;
    if (q0 >= n) return;
    const QueryDesc& d = descs[blockIdx.y];
    const Const& k = v.k;
    const int N = k.N;
    const double px = sp.px, py = sp.py;
    const unsigned char* __restrict__ data = d.data;
    const size_t step = (size_t)d.point_step;
    float x[SAMPLE_ILP], y[SAMPLE_ILP];
#pragma unroll
    for (int u = 0; u < SAMPLE_ILP; ++u) {
        const unsigned q = q0 + u * SAMPLE_THREADS;
        x[u] = y[u] = __uint_as_float(SAMPLE_NAN);
        if (q < n) {
            const unsigned char* p = data + (size_t)q * step;
            x[u] = __ldg(reinterpret_cast<const float*>(p + d.off_x));
            y[u] = __ldg(reinterpret_cast<const float*>(p + d.off_y));
        }
    }
    // per query: its cell a (-1 outside) and, when it interpolates, the neighbours b = (i + si, j), c = (i, j + sj),
    // d = (i + si, j + sj) with their weights (cb = -1: the nearest value)
    int ca[SAMPLE_ILP], cb[SAMPLE_ILP], cc[SAMPLE_ILP], cd[SAMPLE_ILP];
    double wa[SAMPLE_ILP], wb[SAMPLE_ILP], wc[SAMPLE_ILP], wd[SAMPLE_ILP];
#pragma unroll
    for (int u = 0; u < SAMPLE_ILP; ++u) {
        const double dx = (double)x[u], dy = (double)y[u];
        int i, j;
        grid_index(k, px, py, dx, dy, i, j);
        const bool in = grid_inside(k, px, py, dx, dy) && i >= 0 && j >= 0 && i < N && j < N;
        ca[u] = in ? i + j * N : -1;
        cb[u] = cc[u] = cd[u] = -1;
        wa[u] = wb[u] = wc[u] = wd[u] = 0.0;
        if (in && mode == GG_SAMPLE_LINEAR) {
            const double cx = cell_centre(k, px, i), cy = cell_centre(k, py, j);
            const int si = dx >= cx ? -1 : 1, sj = dy >= cy ? -1 : 1;   // i grows toward -x
            if (i + si >= 0 && i + si < N && j + sj >= 0 && j + sj < N) {
                const double tx = __ddiv_rn(fabs(__dsub_rn(dx, cx)), k.res), ty = __ddiv_rn(fabs(__dsub_rn(dy, cy)), k.res);
                const double ux = __dsub_rn(1.0, tx), uy = __dsub_rn(1.0, ty);
                wa[u] = __dmul_rn(ux, uy);
                wb[u] = __dmul_rn(tx, uy);
                wc[u] = __dmul_rn(ux, ty);
                wd[u] = __dmul_rn(tx, ty);
                cb[u] = ca[u] + si;
                cc[u] = ca[u] + sj * N;
                cd[u] = ca[u] + si + sj * N;
            }
        }
    }
    if (d.cell) {
#pragma unroll
        for (int u = 0; u < SAMPLE_ILP; ++u) {
            const unsigned q = q0 + u * SAMPLE_THREADS;
            if (q < n) d.cell[q] = ca[u];
        }
    }
#pragma unroll
    for (int l = 0; l < L_NUM; ++l) {   // static indexing keeps `names` in the parameter bank
        if (l >= names.n) break;
        const int idx = names.idx[l];
        const float* __restrict__ P = v.layer(sp.slot, idx == LAYER_POINTS ? sp.points_layer : idx);
        float fa[SAMPLE_ILP], fb[SAMPLE_ILP], fc[SAMPLE_ILP], fd[SAMPLE_ILP];
#pragma unroll
        for (int u = 0; u < SAMPLE_ILP; ++u) {
            fa[u] = ca[u] >= 0 ? P[ca[u]] : __uint_as_float(SAMPLE_NAN);
            fb[u] = fc[u] = fd[u] = 0.0f;
            if (cb[u] >= 0) {
                fb[u] = P[cb[u]];
                fc[u] = P[cc[u]];
                fd[u] = P[cd[u]];
            }
        }
        float* __restrict__ out = d.dst + (size_t)l * n;
#pragma unroll
        for (int u = 0; u < SAMPLE_ILP; ++u) {
            const unsigned q = q0 + u * SAMPLE_THREADS;
            if (q >= n) break;
            float r = fa[u];
            if (cb[u] >= 0) {
                const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(wa[u], (double)fa[u]), __dmul_rn(wb[u], (double)fb[u])),
                                                     __dmul_rn(wc[u], (double)fc[u])),
                                           __dmul_rn(wd[u], (double)fd[u]));
                r = (float)s;
                if (r != r) r = __uint_as_float(SAMPLE_NAN);
            }
            out[q] = r;
        }
    }
}

// Point classes and heights (gg_point_info_to_device).  Blocks (x, slot): every thread takes PINFO_ILP points of the
// slot's last scan PINFO_THREADS apart (as k_label does), issues their code and z loads up front, then gathers "ground"
// at each point's cell (N^2 floats per slot, L2-resident), then stores codes and heights coalesced.  Heights are
// z - ground[cell] in fp32; an absent point has no cell and gets the quiet NaN 0x7fc00000.
constexpr int PINFO_THREADS = 256, PINFO_ILP = 4;
constexpr uint32_t PINFO_NAN = 0x7fc00000u;

__global__ void __launch_bounds__(PINFO_THREADS) k_point_info(View v, const SlotParams* __restrict__ batch, const PointInfoDest* __restrict__ dests) {
    const SlotParams& sp = batch[blockIdx.y];
    const int n = sp.n_points;
    const int i0 = blockIdx.x * (PINFO_THREADS * PINFO_ILP) + threadIdx.x;
    if (i0 >= n) return;   // the grid covers the largest scan of the batch
    const PointInfoDest d = dests[blockIdx.y];
    const size_t base = (size_t)sp.slot * v.pcap;
    const float* __restrict__ G = v.layer(sp.slot, L_GROUND);
    uint32_t code[PINFO_ILP];
    float z[PINFO_ILP];
#pragma unroll
    for (int u = 0; u < PINFO_ILP; ++u) {
        const int i = i0 + u * PINFO_THREADS;
        code[u] = i < n ? v.code[base + i] : (PC_ABSENT << 24);
        z[u] = (i < n && d.height) ? __uint_as_float(v.zw[base + i].x) : 0.0f;
    }
    if (d.height) {
        float g[PINFO_ILP];
#pragma unroll
        for (int u = 0; u < PINFO_ILP; ++u) g[u] = (code[u] >> 24) != PC_ABSENT ? G[code[u] & 0xffffffu] : 0.0f;
#pragma unroll
        for (int u = 0; u < PINFO_ILP; ++u) {
            const int i = i0 + u * PINFO_THREADS;
            if (i >= n) break;
            d.height[i] = (code[u] >> 24) != PC_ABSENT ? __fsub_rn(z[u], g[u]) : __uint_as_float(PINFO_NAN);
        }
    }
    if (d.codes) {
#pragma unroll
        for (int u = 0; u < PINFO_ILP; ++u) {
            const int i = i0 + u * PINFO_THREADS;
            if (i >= n) break;
            d.codes[i] = code[u];
        }
    }
}

// Poses from device memory (gg_update_poses_from_device).  One thread per staged record; both kernels are tiny and
// exist to keep the host out of the loop, not for throughput.
constexpr int POSE_THREADS = 128;

// A staging entry's records take the slot's device-owned position and / or its device scan pose, and their point count
// from the count tables, after the entry's copy and before the kernels that read them (the same stream).
__global__ void __launch_bounds__(POSE_THREADS) k_stage_poses(PoseTables t, CountTables c, SlotParams* __restrict__ batch, const int* __restrict__ bits,
                                                              int count) {
    const int j = blockIdx.x * POSE_THREADS + threadIdx.x;
    if (j >= count) return;
    const int b = bits[j];
    if (!b) return;
    SlotParams& p = batch[j];
    if (b & POSE_COUNT) {
        // the staged n_points is the scan's capacity: a count outside [0, capacity] runs the scan empty, never clamped
        const int v = c.stored[p.slot];
        const int u = (v >= 0 && v <= p.n_points) ? v : 0;
        p.n_points = u;
        c.last[p.slot] = u;
    }
    if (b & POSE_LAST_COUNT) p.n_points = c.last[p.slot];
    if (b & POSE_POSITION) {
        const double2 q = t.position[p.slot];
        p.px = q.x;
        p.py = q.y;
    }
    if (b & POSE_ORIGIN) {
        const float4 o = t.scan_pose[p.slot];
        p.ox = o.x;
        p.oy = o.y;
        p.oz = o.z;
        p.base_z_f = o.w;
    }
}

// GroundGrid::update's pose step for record j of a roll entry: the cell shift from the caller's odometry position
// (resolve_move, the arithmetic of gg_host.cpp:move_map), the seed row of T_base_from_map, the new position; then
// k_roll_gather / k_roll_commit run on the same records.  A record whose pose is invalid keeps shift 0: the roll
// kernels skip it.  The scan pose is stored as fill_params stages a host one: (float)base_z.
__global__ void __launch_bounds__(POSE_THREADS) k_pose_resolve(double res, PoseTables t, SlotParams* __restrict__ batch, const int* __restrict__ bits,
                                                               int count, DevicePoses in) {
    const int j = blockIdx.x * POSE_THREADS + threadIdx.x;
    if (j >= count) return;
    SlotParams& p = batch[j];
    const int s = p.slot;
    const size_t k = (size_t)p.pos;
    int moved = 0;
    if (in.xy) {
        double px = p.px, py = p.py;
        if (bits[j] & POSE_POSITION) {
            const double2 q = t.position[s];
            px = q.x;
            py = q.y;
        }
        int si = 0, sj = 0;
        moved = resolve_move(res, px, py, in.xy[2 * k], in.xy[2 * k + 1], si, sj);
        p.shift_i = si;
        p.shift_j = sj;
        p.px = px;
        p.py = py;
        const double* T = in.T + 12 * k;
        p.t20 = T[8];
        p.t21 = T[9];
        p.t22 = T[10];
        p.t23 = T[11];
        t.position[s] = make_double2(px, py);
    }
    if (in.origin) t.scan_pose[s] = make_float4(in.origin[3 * k], in.origin[3 * k + 1], in.origin[3 * k + 2], (float)in.base_z[k]);
    if (in.moved) in.moved[k] = moved;
}

// Point counts from device memory (gg_set_point_counts_from_device): record j stores the caller's count of its slot.
// Values are stored as given; k_stage_poses applies the capacity rule when a scan uses them.
__global__ void __launch_bounds__(POSE_THREADS) k_store_counts(CountTables c, const SlotParams* __restrict__ batch, int count,
                                                               const int32_t* __restrict__ dev_n) {
    const int j = blockIdx.x * POSE_THREADS + threadIdx.x;
    if (j >= count) return;
    const SlotParams& p = batch[j];
    c.stored[p.slot] = dev_n[p.pos];
}

// Step plans (gg_step_plan_create): record j of a replay's working UnpackDescs takes its sensor-to-map transform from
// the caller's device memory, read at replay time; the copy is bitwise, so k_unpack_transform computes what it computes
// for the same doubles staged from the host.
__global__ void __launch_bounds__(POSE_THREADS) k_stage_transforms(UnpackDesc* __restrict__ descs, const double* const* __restrict__ T, int count) {
    const int j = blockIdx.x * POSE_THREADS + threadIdx.x;
    if (j >= count) return;
    const double* t = T[j];
    if (!t) return;
    UnpackDesc& d = descs[j];
#pragma unroll
    for (int q = 0; q < 12; ++q) d.T[q] = t[q];
    d.transform = 1;
}

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// GroundGrid::initGroundGrid (src/GroundGrid.cpp:71-75): the value every cell of layer l starts with in a map at height
// z.  ground = z, groundpatch = 1e-7, points = 0, min = 100, max = -100; the per-scan layers start at 0.  k_init_map and
// k_reset_maps both take their values from here.
__device__ __forceinline__ float init_value(int l, float z) {
    switch (l) {
        case L_GROUND: return z;
        case L_GROUNDPATCH: return (float)0.0000001;
        case L_MINH: return 100.0f;
        case L_MAXH: return -100.0f;
        default: return 0.0f;
    }
}

__global__ void __launch_bounds__(256) k_init_map(View v, int slot, float z) {
    const int cell = blockIdx.x * 256 + threadIdx.x;
    if (cell >= v.k.N2) return;
#pragma unroll
    for (int l = 0; l < L_NUM; ++l) {
        if (l >= v.n_layers) break;
        v.layer(slot, l)[cell] = init_value(l, z);
    }
}

int launch_init_map(const View& v, int slot, float z, cudaStream_t st) {
    k_init_map<<<cdiv(v.k.N2, 256), 256, 0, st>>>(v, slot, z);
    return 1;
}

// Map resets from device memory (gg_init_maps_from_device): block (x, j) covers cells [x * RESET_CELLS, (x + 1) *
// RESET_CELLS) of every layer of record j's slot.  A reset of all slots is a pure store stream, so each thread writes
// RESET_VEC consecutive cells per layer (one 16-byte store when N2 % 4 == 0, which keeps every plane 16-byte aligned)
// with all of a slot's layers in flight at once.  A masked-off record costs one mask load per block; its block 0 seeds
// a host-owned position into the table, as k_pose_resolve does, since the host counts the slot's position as
// device-owned afterwards.
constexpr int RESET_THREADS = 256;
constexpr int RESET_VEC = 4;
constexpr int RESET_CELLS = RESET_THREADS * RESET_VEC;

template <bool VEC>
__global__ void __launch_bounds__(RESET_THREADS) k_reset_maps(View v, PoseTables t, const SlotParams* __restrict__ batch, const int* __restrict__ bits,
                                                              const double* __restrict__ xyz, const int32_t* __restrict__ mask) {
    const int j = blockIdx.y;
    const SlotParams& p = batch[j];
    const int k = p.pos;
    const bool first = blockIdx.x == 0 && threadIdx.x == 0;
    if (mask && mask[k] == 0) {
        if (first && !(bits[j] & POSE_POSITION)) t.position[p.slot] = make_double2(p.px, p.py);
        return;
    }
    const int s = p.slot;
    const float z = __double2float_rn(xyz[3 * k + 2]);
    if (first) t.position[s] = make_double2(xyz[3 * k], xyz[3 * k + 1]);
    const int N2 = v.k.N2;
    float* base = v.layer(s, 0);
    const int nl = v.n_layers;
    if (VEC) {
        const int c = blockIdx.x * RESET_CELLS + threadIdx.x * RESET_VEC;
        if (c >= N2) return;
#pragma unroll
        for (int l = 0; l < L_NUM; ++l) {
            if (l >= nl) break;
            const float f = init_value(l, z);
            *reinterpret_cast<float4*>(base + (size_t)l * N2 + c) = make_float4(f, f, f, f);
        }
    } else {
        const int c0 = blockIdx.x * RESET_CELLS + threadIdx.x;
#pragma unroll
        for (int l = 0; l < L_NUM; ++l) {
            if (l >= nl) break;
            const float f = init_value(l, z);
#pragma unroll
            for (int u = 0; u < RESET_VEC; ++u) {
                const int c = c0 + u * RESET_THREADS;
                if (c < N2) base[(size_t)l * N2 + c] = f;
            }
        }
    }
}

struct Mark {
    Profiler* p;
    int id;
    cudaStream_t st;
    Mark(Profiler* p_, int id_, cudaStream_t st_) : p(p_), id(id_), st(st_) {
        if (p) p->begin(id, st);
    }
    ~Mark() {
        if (p) p->end(id, st);
    }
};
#define GG_LAUNCH(id, ...)        \
    do {                          \
        Mark mark__(prof, id, st);\
        __VA_ARGS__;              \
    } while (0)

int launch_roll(const View& v, const SlotParams* batch, int count, cudaStream_t st, Profiler* prof) {
    dim3 grid(cdiv(v.k.N2, 256 * ROLL_ILP), count);
    GG_LAUNCH(K_ROLL_GATHER, k_roll_gather<<<grid, 256, 0, st>>>(v, batch));
    GG_LAUNCH(K_ROLL_COMMIT, k_roll_commit<<<grid, 256, 0, st>>>(v, batch));
    return 2;
}

// patch detection: the TMA-staged tile when the arena has a descriptor (it needs a 16-byte row pitch: N % 4 == 0), else plain loads
static void enqueue_detect(const View& v, const SlotParams* batch, int count, cudaStream_t st, const CUtensorMap* layer_map, int count_layer,
                           bool recompute) {
    if (layer_map)
        k_detect_tma<<<dim3(cdiv(v.k.N, DT_X), cdiv(cdiv(v.k.N, DT_Y), DT_TILES), count), dim3(DT_X, DT_Y), 0, st>>>(v, batch, *layer_map, count_layer,
                                                                                                                     recompute);
    else
        k_detect_ldg<<<dim3(cdiv(v.k.N, DT_X), cdiv(v.k.N, DT_Y), count), dim3(DT_X, DT_Y), 0, st>>>(v, batch, count_layer, recompute);
}

// dynamic shared memory of the skewed / pipelined spiral launch for v
static size_t skew_shm(const View& v) {
    return (size_t)SKEW_RING * v.skew.irr_chunks * sizeof(uint4) + (size_t)SKEW_XCH_DEPTH * v.skew.lanes * sizeof(float2) +
           (size_t)v.skew.irr_max * 9 * sizeof(float2) + (size_t)v.skew.irr_max * sizeof(float) + 16;
}
static size_t pipe_shm(const View& v) {
    return (size_t)((v.levels + 4) & ~3) * sizeof(int) + (size_t)(SPIRAL_PIPE_DIST + 1) * v.spiral_threads * sizeof(float2);
}

int launch_scan_pipeline(const View& v, const SlotParams* batch, int count, int max_points, int stop_after, cudaStream_t st,
                         Profiler* prof, const CUtensorMap* layer_map) {
    int launches = 0;
    const int nb = max(1, cdiv(max_points, RASTER_TILE));

    GG_LAUNCH(K_RASTERIZE, k_rasterize<<<dim3(nb, count), RASTER_THREADS, 0, st>>>(v, batch));
    GG_LAUNCH(K_CELL_TILES, k_cell_tiles<<<dim3(v.cell_tiles, count), CT_THREADS, 0, st>>>(v, batch));
    GG_LAUNCH(K_CELL_PLACE, k_cell_place<<<dim3(v.cell_tiles, count), CT_THREADS, 0, st>>>(v, batch));
    GG_LAUNCH(K_SCATTER, k_scatter<<<dim3(max(1, cdiv(max_points, 256 * SCATTER_ILP)), count), 256, 0, st>>>(v, batch));
    launches += 4;

    if (v.k.full_layers)
        GG_LAUNCH(K_CELL_STATS, k_cell_stats<true><<<dim3(cdiv(v.k.N2, CS_THREADS * 4), count), CS_THREADS, 0, st>>>(v, batch));
    else
        GG_LAUNCH(K_CELL_STATS, k_cell_stats<false><<<dim3(cdiv(v.k.N2, CS_THREADS * 4), count), CS_THREADS, 0, st>>>(v, batch));
    ++launches;
    if (stop_after == 1) return launches;

    GG_LAUNCH(K_DETECT, enqueue_detect(v, batch, count, st, layer_map, L_COUNT, false));
    ++launches;
    if (stop_after == 2) return launches;

    const int threads = v.spiral_threads;
    if (v.skew.sk) {
        const size_t shm = skew_shm(v);
#define GG_SKEW_LAUNCH(T, C)                                                                                                     \
    {                                                                                                                            \
        if (shm > 48 * 1024)   /* large maps: opt in to more dynamic shared memory */                                           \
            cudaFuncSetAttribute(k_spiral_skew<T, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);                    \
        GG_LAUNCH(K_SPIRAL, (k_spiral_skew<T, C><<<count, threads, shm, st>>>(v, batch)));                                       \
    }
        if (threads <= 320)       // small maps: several scans share an SM
            GG_SKEW_LAUNCH(320, 3)
        else if (threads <= 448)
            GG_SKEW_LAUNCH(448, 2)
        else if (threads <= 768)
            GG_SKEW_LAUNCH(768, 1)
        else
            GG_SKEW_LAUNCH(1024, 1)
#undef GG_SKEW_LAUNCH
    } else if (v.spiral_recs) {
        const size_t shm = pipe_shm(v);
#define GG_PIPE_LAUNCH(T)                                                                                                        \
    {                                                                                                                            \
        if (shm > 48 * 1024) cudaFuncSetAttribute(k_spiral_pipe<T, SPIRAL_PIPE_DIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm); \
        GG_LAUNCH(K_SPIRAL, (k_spiral_pipe<T, SPIRAL_PIPE_DIST><<<count, T, shm, st>>>(v, batch)));                             \
    }
        if (threads == 512)
            GG_PIPE_LAUNCH(512)
        else
            GG_PIPE_LAUNCH(1024)
#undef GG_PIPE_LAUNCH
    } else {
        GG_LAUNCH(K_SPIRAL, k_spiral<<<count, SPIRAL_THREADS, 0, st>>>(v, batch));
    }
    ++launches;
    if (stop_after == 3) return launches;

    GG_LAUNCH(K_LABEL, k_label<<<dim3(max(1, cdiv(max_points, 256 * LABEL_ILP)), count), 256, 0, st>>>(v, batch));
    ++launches;
    return launches;
}

// ------------------------------------------------------------------------------------------
// Single phases / single cells on their own: the public per-phase methods of the reference class
// (GroundSegmentation.h:56-62) -- detect_ground_patches, detect_ground_patch<S>, spiral_ground_interpolation,
// interpolate_cell -- for callers that drive the phases themselves.  Same arithmetic as the pipeline kernels.
// ------------------------------------------------------------------------------------------
// GroundSegmentation::interpolate_cell (:445-465) for one cell, in place
__global__ void k_interpolate_cell(View v, const CfgConst kc, int slot, int x, int y) {
    const Const& k = v.k;
    const int N = k.N;
    float* G = v.layer(slot, L_GROUND);
    float* C = v.layer(slot, L_GROUNDPATCH);
    float cc[9], pr[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) {
        const int g = (x - 1 + q % 3) + (y - 1 + q / 3) * N;
        cc[q] = C[g];
        pr[q] = __fmul_rn(cc[q], G[g]);
    }
    const float h = G[x + y * N];
    const float occ = cc[4];
    const float s = __fadd_rn(tree9(cc), FLT_MIN);  // :457
    const float avg = __fdiv_rn(tree9(pr), s);      // :458
    G[x + y * N] = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, occ), avg), __fmul_rn(occ, h));  // :460
    const float fc = (float)(N / 2 - 1);
    const float fx = __fsub_rn((float)x, fc), fy = __fsub_rn((float)y, fc);
    const double d2 = __dmul_rn(__dadd_rn(__dmul_rn((double)fx, (double)fx), __dmul_rn((double)fy, (double)fy)), k.res_sq);
    if (d2 > 12.0) {  // :463
        const double o = (double)occ;
        const double dec = __dsub_rn(o, __ddiv_rn(o, kc.dec_factor));
        C[x + y * N] = (float)((dec < 0.001) ? 0.001 : dec);  // std::max(dec, 0.001)
    }
}

// GroundSegmentation::detect_ground_patch<S> (:343-395) for one cell, reading the layers directly ("points" = count_layer)
template <int S>
__global__ void k_detect_cell(View v, const CfgConst kc, int slot, int i, int j, int count_layer) {
    const Const& k = v.k;
    const int N = k.N, H = S / 2;
    const float* P = v.layer(slot, count_layer);
    const float* V = v.layer(slot, L_VARIANCE);
    const float* M = v.layer(slot, L_MINH);
    float* G = v.layer(slot, L_GROUND);
    float* C = v.layer(slot, L_GROUNDPATCH);
    const int cell = i + j * N;
    auto at = [&](const float* L, int q) { return L[(i - H + q % S) + (j - H + q / S) * N]; };
    const double di = __dsub_rn((double)i, (double)N / 2.0), dj = __dsub_rn((double)j, (double)N / 2.0);
    const float sqdist = (float)__dmul_rn(__dadd_rn(__dmul_rn(di, di), __dmul_rn(dj, dj)), k.res_sq);  // :356
    const float e = v.expected[cell];
    const float psum = TreeSum<0, S * S>::run([&](int q) { return at(P, q); });
    double need = floor(__dmul_rn(__dmul_rn(kc.gp_thresh, (double)S), (double)e));
    need = (need < 3.0) ? 3.0 : need;
    if ((double)psum < need) return;  // :364
    const double a = __dmul_rn((double)sqdist, kc.df_sq);
    const double m = (a < kc.mdf_sq) ? kc.mdf_sq : a;
    const float vt = (float)((kc.mdf10_sq < m) ? kc.mdf10_sq : m);  // :369
    float localmin = at(M, 0);
    for (int q = 1; q < S * S; ++q) {
        const float t = at(M, q);
        localmin = (t < localmin) ? t : localmin;
    }
    const float sumPV = TreeSum<0, S * S>::run([&](int q) { return __fmul_rn(at(P, q), at(V, q)); });
    const float sumPM = TreeSum<0, S * S>::run([&](int q) { return __fmul_rn(at(P, q), at(M, q)); });
    float g = G[cell], c = C[cell];
    if (detect_decide<S>(kc, psum, localmin, sumPV, sumPM, P[cell], V[cell], vt, e, g, c)) {
        G[cell] = g;
        C[cell] = c;
    }
}

int launch_detect_only(const View& v, const SlotParams* batch, int count, cudaStream_t st, Profiler* prof, const CUtensorMap* layer_map,
                       int count_layer, bool recompute) {
    GG_LAUNCH(K_DETECT, enqueue_detect(v, batch, count, st, layer_map, count_layer, recompute));
    return 1;
}

// the plain level-scheduled wavefront on the normal layers (no skewed copy needed)
int launch_spiral_only(const View& v, const SlotParams* batch, int count, cudaStream_t st, Profiler* prof) {
    GG_LAUNCH(K_SPIRAL, k_spiral<<<count, SPIRAL_THREADS, 0, st>>>(v, batch));
    return 1;
}

int launch_interpolate_cell(const View& v, const CfgConst& c, int slot, int x, int y, cudaStream_t st) {
    k_interpolate_cell<<<1, 1, 0, st>>>(v, c, slot, x, y);
    return 1;
}

int launch_detect_cell(const View& v, const CfgConst& c, int slot, int S, int i, int j, int count_layer, cudaStream_t st) {
    if (S == 3)
        k_detect_cell<3><<<1, 1, 0, st>>>(v, c, slot, i, j, count_layer);
    else
        k_detect_cell<5><<<1, 1, 0, st>>>(v, c, slot, i, j, count_layer);
    return 1;
}

int launch_output(const View& v, const SlotParams* batch, const OutDest* dests, int count, int max_points, bool compact, bool write,
                  cudaStream_t st, Profiler* prof) {
    const int nblk = max(1, cdiv(max_points, OUT_TILE));
    int launches = 0;
    if (compact) {
        GG_LAUNCH(K_OUT_COUNT, k_out_count<<<dim3(nblk, count), OUT_TILE, 0, st>>>(v, batch, dests, nblk));
        GG_LAUNCH(K_OUT_SCAN, k_out_scan<<<count, 1024, 0, st>>>(v, batch, dests, nblk));
        launches += 2;
    }
    if (write) {
        GG_LAUNCH(K_OUT_WRITE, k_out_write<<<dim3(nblk, count), OUT_TILE, 0, st>>>(v, batch, dests, nblk));
        ++launches;
    }
    return launches;
}

int launch_layer_copy(const View& v, const SlotParams* batch, int count, const LayerList& names, float* buf, bool import, cudaStream_t st,
                      Profiler* prof) {
    const dim3 grid(cdiv(v.k.N2, LC_THREADS * LC_ILP), count, names.n);
    if (import)
        GG_LAUNCH(K_LAYER_COPY, k_layer_copy<true><<<grid, LC_THREADS, 0, st>>>(v, batch, names, buf));
    else
        GG_LAUNCH(K_LAYER_COPY, k_layer_copy<false><<<grid, LC_THREADS, 0, st>>>(v, batch, names, buf));
    return 1;
}

int launch_unpack(const View& v, const SlotParams* batch, const UnpackDesc* descs, int count, int max_points, cudaStream_t st, Profiler* prof) {
    GG_LAUNCH(K_UNPACK, k_unpack_transform<<<dim3(max(1, cdiv(max_points, 256)), count), 256, 0, st>>>(v, batch, descs));
    return 1;
}

int launch_layer_images(const View& v, const SlotParams* batch, int count, const LayerList& names, int2* partial, unsigned char* dst, float* range,
                        cudaStream_t st, Profiler* prof) {
    const int n_part = cdiv(v.k.N2, IMG_RANGE_CELLS), tiles = cdiv(v.k.N, IMG_TILE);
    GG_LAUNCH(K_LAYER_RANGE, k_layer_range<<<dim3(n_part, count, names.n), IR_THREADS, 0, st>>>(v, batch, names, partial));
    GG_LAUNCH(K_LAYER_IMAGE, k_layer_image<<<dim3(tiles * tiles, count, names.n), dim3(IMG_TILE, IMG_ROWS), 0, st>>>(v, batch, names, partial, n_part, dst, range));
    return 2;
}

int launch_terrain_images(const View& v, const SlotParams* batch, int count, float* dst, cudaStream_t st, Profiler* prof) {
    const int tiles = cdiv(v.k.N, IMG_TILE);
    GG_LAUNCH(K_TERRAIN, k_terrain_image<<<dim3(tiles * tiles, count), dim3(IMG_TILE, IMG_ROWS), 0, st>>>(v, batch, dst));
    return 1;
}

int launch_eval(const View& v, const SlotParams* batch, int count, int max_points, unsigned long long* counts, cudaStream_t st, Profiler* prof) {
    GG_LAUNCH(K_EVAL, k_eval_counts<<<dim3(max(1, cdiv(max_points, EVAL_TILE)), count), EVAL_THREADS, 0, st>>>(v, batch, counts));
    return 1;
}

int launch_sample(const View& v, const SlotParams* batch, const QueryDesc* descs, int count, int max_points, const LayerList& names, int mode,
                  cudaStream_t st, Profiler* prof) {
    constexpr long long per_block = SAMPLE_THREADS * SAMPLE_ILP;   // max_points may be INT32_MAX: no int rounding-up
    const long long blocks = ((long long)max_points + per_block - 1) / per_block;
    const unsigned nb = blocks > 0 ? (unsigned)blocks : 1u;
    GG_LAUNCH(K_SAMPLE, k_sample_layers<<<dim3(nb, count), SAMPLE_THREADS, 0, st>>>(v, batch, descs, names, mode));
    return 1;
}

int launch_point_info(const View& v, const SlotParams* batch, const PointInfoDest* dests, int count, int max_points, cudaStream_t st,
                      Profiler* prof) {
    GG_LAUNCH(K_POINT_INFO, k_point_info<<<dim3(max(1, cdiv(max_points, PINFO_THREADS * PINFO_ILP)), count), PINFO_THREADS, 0, st>>>(v, batch, dests));
    return 1;
}

int launch_stage_poses(const PoseTables& t, const CountTables& c, SlotParams* batch, const int* bits, int count, cudaStream_t st, Profiler* prof) {
    GG_LAUNCH(K_STAGE_POSES, k_stage_poses<<<cdiv(count, POSE_THREADS), POSE_THREADS, 0, st>>>(t, c, batch, bits, count));
    return 1;
}

int launch_store_counts(const CountTables& c, const SlotParams* batch, int count, const int32_t* dev_n, cudaStream_t st, Profiler* prof) {
    GG_LAUNCH(K_STORE_COUNTS, k_store_counts<<<cdiv(count, POSE_THREADS), POSE_THREADS, 0, st>>>(c, batch, count, dev_n));
    return 1;
}

int launch_stage_transforms(UnpackDesc* descs, const double* const* T, int count, cudaStream_t st) {
    k_stage_transforms<<<cdiv(count, POSE_THREADS), POSE_THREADS, 0, st>>>(descs, T, count);
    return 1;
}

int prepare_scan_pipeline(const View& v) {
    const int threads = v.spiral_threads;
    cudaError_t e = cudaSuccess;
    if (v.skew.sk) {
        const size_t shm = skew_shm(v);
        if (shm > 48 * 1024) {
            if (threads <= 320)
                e = cudaFuncSetAttribute(k_spiral_skew<320, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
            else if (threads <= 448)
                e = cudaFuncSetAttribute(k_spiral_skew<448, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
            else if (threads <= 768)
                e = cudaFuncSetAttribute(k_spiral_skew<768, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
            else
                e = cudaFuncSetAttribute(k_spiral_skew<1024, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
        }
    } else if (v.spiral_recs) {
        const size_t shm = pipe_shm(v);
        if (shm > 48 * 1024)
            e = threads == 512 ? cudaFuncSetAttribute(k_spiral_pipe<512, SPIRAL_PIPE_DIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm)
                               : cudaFuncSetAttribute(k_spiral_pipe<1024, SPIRAL_PIPE_DIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm);
    }
    return e == cudaSuccess ? 0 : -1;
}

int launch_pose_resolve(const View& v, const PoseTables& t, SlotParams* batch, const int* bits, int count, const DevicePoses& in, cudaStream_t st,
                        Profiler* prof) {
    GG_LAUNCH(K_POSE_RESOLVE, k_pose_resolve<<<cdiv(count, POSE_THREADS), POSE_THREADS, 0, st>>>(v.k.res, t, batch, bits, count, in));
    return 1;
}

int launch_reset_maps(const View& v, const PoseTables& t, const SlotParams* batch, const int* bits, int count, const double* xyz, const int32_t* mask,
                      cudaStream_t st, Profiler* prof) {
    const dim3 grid(cdiv(v.k.N2, RESET_CELLS), count);
    if (v.k.N2 % RESET_VEC == 0)
        GG_LAUNCH(K_RESET_MAPS, k_reset_maps<true><<<grid, RESET_THREADS, 0, st>>>(v, t, batch, bits, xyz, mask));
    else
        GG_LAUNCH(K_RESET_MAPS, k_reset_maps<false><<<grid, RESET_THREADS, 0, st>>>(v, t, batch, bits, xyz, mask));
    return 1;
}

}  // namespace gg
