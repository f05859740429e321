// =====================================================================================
// TEST INFRASTRUCTURE ONLY.  CPU oracle for the GroundGrid per-scan hot path.
//
// This file is a CPU restatement (C++17, no FMA contraction, no fast-math) of the
// reference algorithm, used ONLY as the checker in tests/, in
// __graft_entry__.smoke(), and as the timed CPU arm of bench.py (cpu_baseline and
// --impl reference).  The product (groundgrid_b200/csrc, groundgrid_b200/host) never
// includes, links or calls anything in oracle/.
//
// PINNED BY THE REFERENCE ITSELF: the reference repository has no tests, golden vectors or fixtures (SURVEY.md
// section 4 / 8c), but its two source files of this path compile unmodified against CPU stand-ins
// (oracle/build_ref.py -> oracle/_ref/libgg_ref.so, see oracle/ref_harness.cpp).  tests/test_oracle_vs_ref.py
// demands that this port and that library agree bit for bit (every layer, label, output position, map roll) on the
// BASELINE configurations, rolling streams with outliers, random geometries / configs; tests/golden/ holds vectors
// produced by the reference library.  What the stand-ins restate from published third-party sources -- Eigen 3.3.7's
// reduction order, grid_map_core 1.6.x geometry, tf2's point transform -- is restated here in the same way
// (eigen_redux.hpp, gridmap_semantics.hpp).  Parity is DEFINED as the reference's thread_count = 1 execution (the
// shipped thread_count = 8 has data races, GroundSegmentation.cpp:99-109 vs :234,282-309).
//
// Build: see oracle/Makefile  (g++ -O3 -DNDEBUG -std=c++17 -ffp-contract=off).
// =====================================================================================
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <limits>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "eigen_redux.hpp"
#include "gridmap_semantics.hpp"

namespace ggo {

// include/velodyne_pointcloud/point_types.h:27-33 -- PointXYZIR, 16-byte aligned, sizeof == 32.
struct alignas(16) Point {
    float x, y, z, pad0;
    float intensity;
    uint16_t ring;
    uint16_t pad1;
    float pad2, pad3;
};
static_assert(sizeof(Point) == 32, "PointXYZIR layout");

// cfg/GroundGrid.cfg:8-21 (same order, same defaults).
struct Config {
    int point_count_cell_variance_threshold = 10;
    int max_ring = 1024;
    double groundpatch_detection_minimum_threshold = 0.01;  // declared, never read
    double distance_factor = 0.0001;
    double minimum_distance_factor = 0.0005;
    double miminum_point_height_threshold = 0.3;
    double minimum_point_height_obstacle_threshold = 0.1;
    double outlier_tolerance = 0.1;
    double ground_patch_detection_minimum_point_count_threshold = 0.25;
    double patch_size_change_distance = 20.0;
    double occupied_cells_decrease_factor = 5.0;
    double occupied_cells_point_count_factor = 20.0;
    double min_outlier_detection_ground_confidence = 1.25;
    int thread_count = 8;
};

using Layer = std::vector<float>;
using IndexedCell = std::pair<size_t, std::pair<int, int>>;  // (point index, (row, col))

class Oracle {
  public:
    Config cfg;
    MapGeometry geo;
    bool have_map = false;
    float resolution_f = 0.f;
    double dimension_m = 0.0;
    int n = 0;  // cells per side
    Layer expected;  // expectedPoints table
    // Fixed layer slots (the reference binds static references once, GroundSegmentation.cpp:76-78,
    // 203-213; a name lookup per cell would be an unfair slowdown of the CPU baseline).
    static constexpr int kNumLayers = 11;
    static const char* layer_name(int k) {
        static const char* names[kNumLayers] = {"points", "ground", "groundpatch", "minGroundHeight", "maxGroundHeight",
                                                "groundCandidates", "planeDist", "m2", "meanVariance", "pointsRaw", "variance"};
        return names[k];
    }
    Layer layers[kNumLayers];
    bool present[kNumLayers] = {false};
    int find_layer(const char* name) const {
        for (int k = 0; k < kNumLayers; ++k)
            if (std::strcmp(name, layer_name(k)) == 0) return k;
        return -1;
    }

    // include/groundgrid/GroundSegmentation.h:69-70
    const float verticalPointAngDist = 0.00174532925 * 2;
    const float minDistSquared = 12.0f;

    Layer& L(const char* name) {
        const int k = find_layer(name);
        present[k] = true;
        return layers[k];
    }
    // Layer bindings for the per-cell functions (the reference's function-local statics).
    struct Hot {
        float *ground = nullptr, *groundpatch = nullptr, *variance = nullptr, *minGroundHeight = nullptr, *points = nullptr;
    } hot;
    void bind_hot() {
        hot.ground = L("ground").data();
        hot.groundpatch = L("groundpatch").data();
        hot.variance = present[find_layer("variance")] ? L("variance").data() : nullptr;
        hot.minGroundHeight = L("minGroundHeight").data();
        hot.points = L("points").data();
    }

    // GroundSegmentation::init -- src/GroundSegmentation.cpp:37-48
    void init(double dimension, float resolution) {
        dimension_m = dimension;
        resolution_f = resolution;
        const size_t cellCount = std::round(static_cast<float>(dimension) / resolution);
        n = static_cast<int>(cellCount);
        expected.assign(cellCount * cellCount, 0.f);
        for (size_t i = 0; i < cellCount; ++i)
            for (size_t j = 0; j < cellCount; ++j) {
                const float dist = std::hypot(i - cellCount / 2.0, j - cellCount / 2.0);
                expected[i + j * cellCount] = std::atan(1 / dist) / verticalPointAngDist;
            }
    }

    // GroundGrid::initGroundGrid -- src/GroundGrid.cpp:50-80
    void init_map(double x, double y, double z) {
        set_geometry(geo, static_cast<double>(static_cast<float>(dimension_m)), static_cast<double>(resolution_f), x, y);
        const size_t cells = static_cast<size_t>(geo.n) * geo.n;
        for (int k = 0; k < kNumLayers; ++k) {
            layers[k].clear();
            present[k] = false;
        }
        L("points").assign(cells, 0.f);
        L("ground").assign(cells, static_cast<float>(z));
        L("groundpatch").assign(cells, static_cast<float>(0.0000001));
        L("minGroundHeight").assign(cells, static_cast<float>(100.0));
        L("maxGroundHeight").assign(cells, static_cast<float>(-100.0));
        have_map = true;
    }

    // GroundGrid::update -- src/GroundGrid.cpp:83-147.  T = row-major 3x4 [R|t] of
    // lookupTransform("base_link", "map") (tf2::doTransform: R*p + t in fp64).
    // Returns 1 if the map moved.
    int update(double x, double y, const double* T) {
        if (!have_map) return -1;
        int si = 0, sj = 0;
        move_shift(geo, x, y, si, sj);
        if (si == 0 && sj == 0) return 0;
        const int N = geo.n;
        const float nanv = std::numeric_limits<float>::quiet_NaN();
        for (int k = 0; k < kNumLayers; ++k) {
            if (!present[k]) continue;
            Layer& src = layers[k];
            Layer dst(src.size(), nanv);  // move(): exposed strips are cleared to NaN in all layers
            for (int c = 0; c < N; ++c) {
                const int oc = c + sj;
                if (oc < 0 || oc >= N) continue;
                for (int r = 0; r < N; ++r) {
                    const int orr = r + si;
                    if (orr < 0 || orr >= N) continue;
                    dst[r + c * N] = src[orr + oc * N];
                }
            }
            src.swap(dst);
        }
        Layer& G = L("ground");
        Layer& C = L("groundpatch");
        for (int c = 0; c < N; ++c)
            for (int r = 0; r < N; ++r) {
                const bool fresh = (r + si < 0 || r + si >= N || c + sj < 0 || c + sj >= N);
                if (!fresh) continue;
                double px, py;
                get_position(geo, r, c, px, py);
                // tf2::Transform * Vector3: row.dot(v) + origin, v = (px, py, 0)
                const double tz = (T[8] * px + T[9] * py + T[10] * 0.0) + T[11];
                G[r + c * N] = static_cast<float>(-tz);
                C[r + c * N] = 0.0f;
            }
        return 1;
    }

    // GroundSegmentation::insert_cloud -- src/GroundSegmentation.cpp:200-311
    void insert_cloud(const Point* cloud, size_t start, size_t end, const Point& origin,
                      std::vector<IndexedCell>& point_index, std::vector<IndexedCell>& ignored,
                      std::vector<size_t>& outliers) {
        const float* ggp = L("groundpatch").data();
        float* gpr = L("pointsRaw").data();
        float* gpl = L("points").data();
        const float* ggl = L("ground").data();
        float* gmg = L("groundCandidates").data();
        float* gmm = L("meanVariance").data();
        float* gmx = L("maxGroundHeight").data();
        float* gmi = L("minGroundHeight").data();
        float* gmd = L("planeDist").data();
        float* gm2 = L("m2").data();
        const int N = geo.n;
        point_index.reserve(end - start);

        for (size_t i = start; i < end; ++i) {
            const Point& point = cloud[i];
            const double posx = point.x, posy = point.y;
            const float sqdist = std::pow(point.x - origin.x, 2.0) + std::pow(point.y - origin.y, 2.0);
            bool toSkip = false;

            int gi0, gi1;
            get_index(geo, posx, posy, gi0, gi1);
            if (!is_inside(geo, posx, posy)) continue;
            // The reference would index out of bounds here (UB) if rounding put an inside
            // position on index n; the oracle defines such points as dropped.
            if (gi0 < 0 || gi1 < 0 || gi0 >= N || gi1 >= N) continue;
            const size_t cell = static_cast<size_t>(gi0) + static_cast<size_t>(gi1) * N;

            gpr[cell] += 1.0f;  // :234

            if (point.ring > cfg.max_ring || sqdist < minDistSquared) {  // :237-240
                ignored.push_back({i, {gi0, gi1}});
                continue;
            }

            // Outlier detection test, :243-275
            const float oldgroundheight = ggl[cell];
            if (point.z < oldgroundheight - 0.2) {
                float vx = point.x - origin.x;
                float vy = point.y - origin.y;
                float vz = point.z - origin.z;
                float len = std::sqrt(std::pow(vx, 2.0f) + std::pow(vy, 2.0f) + std::pow(vz, 2.0f));
                vx /= len;
                vy /= len;
                vz /= len;
                for (int step = 3;
                     (std::pow(step * vx, 2.0) + std::pow(step * vy, 2.0) + std::pow(step * vz, 2.0)) < std::pow(len, 2.0) &&
                     vz < -0.01f;
                     ++step) {
                    int ix, iy;
                    get_index(geo, step * vx + origin.x, step * vy + origin.y, ix, iy);
                    if (ix <= 0 || iy <= 0 || ix >= N - 1 || iy >= N - 1) continue;
                    const float bsum = block_sum<3>(ggp, N, std::max(ix - 1, 2), std::max(iy - 1, 2));
                    if (bsum > cfg.min_outlier_detection_ground_confidence && ggp[ix + iy * N] > 0.01f &&
                        ggl[ix + iy * N] >= step * vz + origin.z + cfg.outlier_tolerance) {
                        outliers.push_back(i);
                        toSkip = true;
                        break;
                    }
                }
            }
            if (toSkip) continue;

            // :282-309
            float& groundheight = gmg[cell];
            float& mean = gmm[cell];
            float planeDist = 0.0;
            point_index.push_back({i, {gi0, gi1}});
            float& points = gpl[cell];
            float& maxHeight = gmx[cell];
            float& minHeight = gmi[cell];
            float& planeDistMap = gmd[cell];
            float& m2 = gm2[cell];

            planeDist = point.z - origin.z;
            groundheight = (point.z + points * groundheight) / (points + 1.0);

            if (mean == 0.0) mean = planeDist;
            if (!std::isnan(planeDist)) {
                float delta = planeDist - mean;
                mean += delta / (points + 1);
                planeDistMap = (planeDist + points * planeDistMap) / (points + 1.0);
                m2 += delta * (planeDist - mean);
            }
            maxHeight = std::max(maxHeight, point.z);
            minHeight = std::min(minHeight, point.z - 0.0001f);
            points += 1.0;
        }
    }

    // GroundSegmentation::detect_ground_patch<S> -- src/GroundSegmentation.cpp:343-395
    template <int S>
    void detect_ground_patch(size_t i, size_t j) {
        float* ggl = hot.ground;
        float* ggp = hot.groundpatch;
        const float* ggv = hot.variance;
        const float* gmi = hot.minGroundHeight;
        const float* gpl = hot.points;
        const int N = geo.n;
        const float resolution = geo.res;
        const int center_idx = std::floor(S / 2);
        const int r0 = static_cast<int>(i) - center_idx, c0 = static_cast<int>(j) - center_idx;

        const float sqdist = (std::pow(i - (N / 2.0), 2.0) + std::pow(j - (N / 2.0), 2.0)) * std::pow(resolution, 2.0);
        const int patchSize = S;
        const float expectedPointCountperLaserperCell = expected[i + j * N];
        const float pointsblockSum = block_sum<S>(gpl, N, r0, c0);
        float& oldConfidence = ggp[i + j * N];
        float& oldGroundheight = ggl[i + j * N];

        if (pointsblockSum <
            std::max(std::floor(cfg.ground_patch_detection_minimum_point_count_threshold * patchSize * expectedPointCountperLaserperCell), 3.0))
            return;

        const float varThresholdsq =
            std::min(std::max(sqdist * std::pow(cfg.distance_factor, 2.0), std::pow(cfg.minimum_distance_factor, 2.0)),
                     std::pow(cfg.minimum_distance_factor * 10, 2.0));
        const float variance = ggv[i + j * N];
        const float localmin = block_min<S>(gmi, N, r0, c0);
        const float centerPoints = gpl[i + j * N];
        const float maxVar = centerPoints >= cfg.point_count_cell_variance_threshold
                                 ? variance
                                 : block_dot<S>(gpl, ggv, N, r0, c0) / pointsblockSum;
        const float groundlevel = block_dot<S>(gpl, gmi, N, r0, c0) / pointsblockSum;
        const float groundDiff = std::max((groundlevel - oldGroundheight) * (2.0f * oldConfidence), 1.0f);

        if (oldConfidence > 0.5 && groundlevel >= oldGroundheight + cfg.outlier_tolerance) return;

        if (varThresholdsq > std::pow(maxVar, 2.0) && maxVar > 0 &&
            pointsblockSum > (groundDiff * expectedPointCountperLaserperCell * patchSize) *
                                 cfg.ground_patch_detection_minimum_point_count_threshold) {
            const float newConfidence = std::min(pointsblockSum / cfg.occupied_cells_point_count_factor, 1.0);
            oldGroundheight = (groundlevel * newConfidence + oldConfidence * oldGroundheight * 2) / (newConfidence + oldConfidence * 2);
            oldConfidence = std::min((pointsblockSum / (cfg.occupied_cells_point_count_factor * 2.0f) + oldConfidence) / 2.0, 1.0);
        } else if (localmin < oldGroundheight) {
            oldGroundheight = localmin;
            oldConfidence = std::min(oldConfidence + 0.1f, 0.5f);
        }
    }

    void compute_variance() {  // :323
        const Layer& gm2 = L("m2");
        const Layer& gpl = L("points");
        Layer& ggv = L("variance");
        for (size_t k = 0; k < ggv.size(); ++k) ggv[k] = gm2[k] / (gpl[k] + std::numeric_limits<float>::min());
    }

    // GroundSegmentation::detect_ground_patches -- src/GroundSegmentation.cpp:314-340
    void detect_ground_patches(unsigned short section) {
        compute_variance();
        const int N = geo.n;
        const float resolution = geo.res;
        const int cols = N, rows = N;
        int cols_start = 2 + section % 2 * (cols / 2 - 2);
        int rows_start = section >= 2 ? rows / 2 : 2;
        int cols_end = (cols) / 2 + section % 2 * (cols / 2 - 2);
        int rows_end = section >= 2 ? rows - 2 : (rows) / 2;
        for (int i = cols_start; i < cols_end; ++i)
            for (int j = rows_start; j < rows_end; ++j) {
                const float sqdist = (std::pow(i - (N / 2.0), 2.0) + std::pow(j - (N / 2.0), 2.0)) * std::pow(resolution, 2.0);
                if (sqdist <= std::pow(cfg.patch_size_change_distance, 2.0))
                    detect_ground_patch<3>(i, j);
                else
                    detect_ground_patch<5>(i, j);
            }
    }

    // GroundSegmentation::interpolate_cell -- src/GroundSegmentation.cpp:445-465
    void interpolate_cell(size_t x, size_t y) {
        const int N = geo.n;
        const int center_idx = N / 2 - 1;
        float* gvl = hot.groundpatch;
        float* ggl = hot.ground;
        float& height = ggl[x + y * N];
        float& occupied = gvl[x + y * N];
        const int r0 = static_cast<int>(x) - 1, c0 = static_cast<int>(y) - 1;
        const float gvlSum = block_sum<3>(gvl, N, r0, c0) + std::numeric_limits<float>::min();
        const float avg = block_dot<3>(gvl, ggl, N, r0, c0) / gvlSum;
        height = (1.0f - occupied) * avg + occupied * height;
        if ((std::pow((float)x - center_idx, 2.0) + std::pow((float)y - center_idx, 2.0)) * std::pow(geo.res, 2.0f) > minDistSquared)
            occupied = std::max(occupied - occupied / cfg.occupied_cells_decrease_factor, 0.001);
    }

    // GroundSegmentation::spiral_ground_interpolation -- src/GroundSegmentation.cpp:398-441
    void spiral_ground_interpolation(double base_z) {
        bind_hot();
        const int N = geo.n;
        const int center_idx = N / 2 - 1;
        L("groundpatch")[center_idx + center_idx * N] = 1.0f;
        L("ground")[center_idx + center_idx * N] = base_z;  // z of mapToBase * (0,0,0)
        for (int i = center_idx - 1; i >= 1; --i) {
            int rectangle_pos = i;
            int side_length = (center_idx - rectangle_pos) * 2;
            for (short side = 0; side < 2; ++side)
                for (int pos = rectangle_pos; pos < rectangle_pos + side_length; ++pos) {
                    const int x = side % 2 ? pos : rectangle_pos;
                    const int y = side % 2 ? rectangle_pos : pos;
                    interpolate_cell(x, y);
                }
            rectangle_pos += side_length;
            for (short side = 0; side < 2; ++side)
                for (int pos = rectangle_pos; pos >= rectangle_pos - side_length; --pos) {
                    int x = side % 2 ? pos : rectangle_pos;
                    int y = side % 2 ? rectangle_pos : pos;
                    interpolate_cell(x, y);
                }
        }
    }

    void reset_scan_layers() {  // src/GroundSegmentation.cpp:61-75
        const size_t cells = static_cast<size_t>(geo.n) * geo.n;
        for (const char* nm : {"groundCandidates", "planeDist", "m2", "meanVariance", "pointsRaw", "variance", "points"})
            L(nm).assign(cells, 0.f);
        L("minGroundHeight").assign(cells, std::numeric_limits<float>::max());
        L("maxGroundHeight").assign(cells, std::numeric_limits<float>::min());
    }

    // GroundSegmentation::filter_cloud -- src/GroundSegmentation.cpp:50-197.
    // stop_after: 0 = whole call, 1 = after rasterisation, 2 = after patch detection,
    // 3 = after spiral interpolation (for per-phase parity tests; layers can then be read).
    // threads <= 0 -> cfg.thread_count.  labels[i] = 0 (absent from output), 49 or 99.
    size_t filter_cloud(const Point* cloud, size_t npts, const Point& origin, double base_z, int threads,
                        int stop_after, uint8_t* labels, Point* out_cloud, uint32_t* out_index, uint8_t* classes = nullptr) {
        reset_scan_layers();
        bind_hot();
        const int N = geo.n;
        const size_t threadcount = threads > 0 ? threads : cfg.thread_count;

        std::vector<IndexedCell> point_index;
        std::vector<std::vector<IndexedCell>> point_index_list(threadcount), ignored_list(threadcount);
        std::vector<size_t> outliers;
        std::vector<std::vector<size_t>> outliers_list(threadcount);
        std::vector<IndexedCell> ignored;

        if (threadcount == 1) {
            insert_cloud(cloud, 0, npts, origin, point_index_list[0], ignored_list[0], outliers_list[0]);
        } else {
            std::vector<std::thread> workers;
            for (size_t i = 0; i < threadcount; ++i) {
                const size_t start = std::floor((i * npts) / threadcount);
                const size_t end = std::ceil(((i + 1) * npts) / threadcount);
                workers.emplace_back([&, i, start, end] {
                    insert_cloud(cloud, start, end, origin, point_index_list[i], ignored_list[i], outliers_list[i]);
                });
            }
            for (auto& w : workers) w.join();
        }
        for (auto& part : point_index_list) point_index.insert(point_index.end(), part.begin(), part.end());
        for (auto& part : outliers_list) outliers.insert(outliers.end(), part.begin(), part.end());
        for (auto& part : ignored_list) ignored.insert(ignored.end(), part.begin(), part.end());
        if (labels) std::memset(labels, 0, npts);
        if (classes) {  // the point classes of the CUDA path (gg_get_point_classes >> 24): 0 outside, 1 / 2 kept, 3 / 4 ignored
                        // (inner / border cell, :167-168), 5 outlier
            std::memset(classes, 0, npts);
            auto mark = [&](const std::vector<IndexedCell>& part, uint8_t inner) {
                for (const IndexedCell& e : part)
                    classes[e.first] = (N <= e.second.first + 3 || N <= e.second.second + 3) ? inner + 1 : inner;
            };
            mark(point_index, 1);
            mark(ignored, 3);
            for (size_t i : outliers) classes[i] = 5;
        }
        if (stop_after == 1) return 0;

        if (threads == 1) {
            // sections are disjoint and each cell only writes its own G/C -> order-free
            for (unsigned short s = 0; s < 4; ++s) detect_ground_patches(s);
        } else {
            std::vector<std::thread> workers;
            for (unsigned short s = 0; s < 4; ++s) workers.emplace_back([this, s] { detect_ground_patches(s); });
            for (auto& w : workers) w.join();
        }
        if (stop_after == 2) return 0;

        spiral_ground_interpolation(base_z);
        if (stop_after == 3) return 0;

        // label loop, :146-196
        Layer& gpl = L("points");
        std::fill(gpl.begin(), gpl.end(), 0.0f);
        const Layer& ggl = L("ground");
        const Layer& ggv = L("variance");
        point_index.insert(point_index.end(), ignored.begin(), ignored.end());

        const double min_dist_fac = cfg.minimum_distance_factor * 5;
        const double min_point_height_thres = cfg.miminum_point_height_threshold;
        const double min_point_height_obs_thres = cfg.minimum_point_height_obstacle_threshold;
        size_t nout = 0;
        auto emit = [&](size_t idx, float value) {
            if (labels) labels[idx] = static_cast<uint8_t>(value);
            if (out_cloud) {
                out_cloud[nout] = cloud[idx];
                out_cloud[nout].intensity = value;
            }
            if (out_index) out_index[nout] = static_cast<uint32_t>(idx);
            ++nout;
        };
        for (const IndexedCell& entry : point_index) {
            const Point& point = cloud[entry.first];
            const int g0 = entry.second.first, g1 = entry.second.second;
            const double groundheight = ggl[g0 + static_cast<size_t>(g1) * N];
            const float variance = ggv[g0 + static_cast<size_t>(g1) * N];
            if (N <= g0 + 3 || N <= g1 + 3) continue;
            const float dist = std::hypot(point.x - origin.x, point.y - origin.y);
            const double tolerance =
                std::max(std::min((min_dist_fac * dist) / variance * min_point_height_thres, min_point_height_thres), min_point_height_obs_thres);
            if (tolerance + groundheight < point.z) {
                emit(entry.first, 99);
                gpl[g0 + static_cast<size_t>(g1) * N] += 1.0f;
            } else {
                emit(entry.first, 49);
            }
        }
        for (size_t i : outliers) emit(i, 49);
        return nout;
    }
};

}  // namespace ggo

// ------------------------------------------------------------------------------------
// C entry points for ctypes (tests / bench cpu arm only).
// ------------------------------------------------------------------------------------
extern "C" {

void* ggo_create(double dimension_m, float resolution) {
    auto* o = new ggo::Oracle();
    o->init(dimension_m, resolution);
    return o;
}
void ggo_destroy(void* h) { delete static_cast<ggo::Oracle*>(h); }
int ggo_cells_per_side(void* h) { return static_cast<ggo::Oracle*>(h)->n; }
void ggo_set_config(void* h, const ggo::Config* c) { static_cast<ggo::Oracle*>(h)->cfg = *c; }
void ggo_get_config(void* h, ggo::Config* c) { *c = static_cast<ggo::Oracle*>(h)->cfg; }
void ggo_init_map(void* h, double x, double y, double z) { static_cast<ggo::Oracle*>(h)->init_map(x, y, z); }
int ggo_update(void* h, double x, double y, const double* T) { return static_cast<ggo::Oracle*>(h)->update(x, y, T); }
void ggo_get_position(void* h, double* xy) {
    auto* o = static_cast<ggo::Oracle*>(h);
    xy[0] = o->geo.px;
    xy[1] = o->geo.py;
}
int ggo_get_expected(void* h, float* dst) {
    auto* o = static_cast<ggo::Oracle*>(h);
    std::memcpy(dst, o->expected.data(), o->expected.size() * sizeof(float));
    return 0;
}
int ggo_get_layer(void* h, const char* name, float* dst) {
    auto* o = static_cast<ggo::Oracle*>(h);
    const int k = o->find_layer(name);
    if (k < 0 || !o->present[k]) return -1;
    std::memcpy(dst, o->layers[k].data(), o->layers[k].size() * sizeof(float));
    return 0;
}
int ggo_set_layer(void* h, const char* name, const float* src) {
    auto* o = static_cast<ggo::Oracle*>(h);
    const int k = o->find_layer(name);
    if (k < 0 || !o->present[k]) return -1;
    std::memcpy(o->layers[k].data(), src, o->layers[k].size() * sizeof(float));
    return 0;
}
// returns number of points in the output cloud; labels (npts bytes), out_cloud (npts records),
// out_index (npts u32: input index of every output point, reference order) and classes (npts bytes: the class of
// every input point, as filter_cloud above numbers them) may be NULL.
long ggo_filter_cloud(void* h, const void* pts, size_t npts, const float* origin3, double base_z, int threads,
                      int stop_after, uint8_t* labels, void* out_cloud, uint32_t* out_index, uint8_t* classes) {
    auto* o = static_cast<ggo::Oracle*>(h);
    if (!o->have_map) return -1;
    ggo::Point origin{};
    origin.x = origin3[0];
    origin.y = origin3[1];
    origin.z = origin3[2];
    return static_cast<long>(o->filter_cloud(static_cast<const ggo::Point*>(pts), npts, origin, base_z, threads, stop_after,
                                             labels, static_cast<ggo::Point*>(out_cloud), out_index, classes));
}
// Isolated pieces for known-answer tests.
void ggo_interpolate_cell(void* h, int x, int y) {
    static_cast<ggo::Oracle*>(h)->bind_hot();
    static_cast<ggo::Oracle*>(h)->interpolate_cell(x, y);
}
void ggo_spiral(void* h, double base_z) { static_cast<ggo::Oracle*>(h)->spiral_ground_interpolation(base_z); }
// detect_ground_patches for all four sections, each starting with the variance recompute of :323, as filter_cloud
// calls them; -1 if the map has no "m2" / "variance" layer yet (the reference's map["m2"] would throw)
int ggo_detect_ground_patches(void* h) {
    auto* o = static_cast<ggo::Oracle*>(h);
    if (!o->have_map || !o->present[o->find_layer("m2")] || !o->present[o->find_layer("variance")]) return -1;
    o->bind_hot();
    for (unsigned short s = 0; s < 4; ++s) o->detect_ground_patches(s);
    return 0;
}
// detect_ground_patch<S>(map, i, j) alone: reads "variance" as stored (no recompute)
int ggo_detect_ground_patch(void* h, int S, int i, int j) {
    auto* o = static_cast<ggo::Oracle*>(h);
    if (!o->have_map || !o->present[o->find_layer("variance")] || (S != 3 && S != 5)) return -1;
    o->bind_hot();
    if (S == 3)
        o->detect_ground_patch<3>(i, j);
    else
        o->detect_ground_patch<5>(i, j);
    return 0;
}
// grid_map::GridMap::add(name, value): a new layer, or an existing one overwritten, with the constant value
int ggo_add_layer(void* h, const char* name, double value) {
    auto* o = static_cast<ggo::Oracle*>(h);
    const int k = o->find_layer(name);
    if (k < 0 || !o->have_map) return -1;
    o->L(name).assign(static_cast<size_t>(o->geo.n) * o->geo.n, static_cast<float>(value));
    return 0;
}
void ggo_grid_index(void* h, double x, double y, int* idx2, int* inside) {
    auto* o = static_cast<ggo::Oracle*>(h);
    ggo::get_index(o->geo, x, y, idx2[0], idx2[1]);
    *inside = ggo::is_inside(o->geo, x, y) ? 1 : 0;
}
void ggo_cell_position(void* h, int i, int j, double* xy) {
    auto* o = static_cast<ggo::Oracle*>(h);
    ggo::get_position(o->geo, i, j, xy[0], xy[1]);
}
float ggo_block_sum3(const float* m, int n, int r0, int c0) { return ggo::block_sum<3>(m, n, r0, c0); }
float ggo_block_sum5(const float* m, int n, int r0, int c0) { return ggo::block_sum<5>(m, n, r0, c0); }
}
