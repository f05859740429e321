// Host-side (no CUDA) pieces of the library: expectedPoints table, config-derived constants,
// the map-move arithmetic and the wavefront schedule of the spiral interpolation.  They are
// exported with a gg_host_ prefix so the CPU test-suite can exercise them without a GPU.
#include <immintrin.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <thread>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <sched.h>

#include "gg_host.h"

namespace gg {

// GroundSegmentation::init (src/GroundSegmentation.cpp:37-48).  Built on the host with the
// platform libm (hypot / atanf), exactly like the reference, then uploaded once.
int cells_per_side(double dimension_m, float resolution) {
    return (int)std::round((float)dimension_m / resolution);
}

void build_expected_points(int n, std::vector<float>& table) {
    const float vertical_point_ang_dist = 0.00174532925 * 2;  // GroundSegmentation.h:69
    table.assign((size_t)n * n, 0.0f);
    const size_t cells = (size_t)n;
    for (size_t i = 0; i < cells; ++i)
        for (size_t j = 0; j < cells; ++j) {
            const float dist = std::hypot(i - cells / 2.0, j - cells / 2.0);
            table[i + j * cells] = std::atan(1 / dist) / vertical_point_ang_dist;
        }
}

// grid_map::GridMap::setGeometry and the geometry constants the kernels need; squares are written as
// x * x, which is what the reference's compiler emits for std::pow(x, 2.0).
void derive_geometry(double dimension_m, float resolution, unsigned flags, Const& k) {
    const double res = (double)resolution;
    const int n = (int)std::round((double)(float)dimension_m / res);
    k.N = n;
    k.N2 = n * n;
    k.full_layers = (flags & GG_FLAG_FULL_LAYERS) ? 1 : 0;
    k.res_f = (float)res;
    k.res = res;
    k.rres = 1.0 / res;
    k.len = (double)n * res;
    k.half = 0.5 * k.len;
    k.res_sq = (double)k.res_f * (double)k.res_f;
}

void ConfigRegistry::reset(int n_slots, const CfgConst& k) {
    for (Variant& v : vars_) v.refs = 0;
    if (vars_.empty()) vars_.push_back(Variant{});
    vars_[0].k = k;
    vars_[0].refs = n_slots;
    slot_var_.assign((size_t)n_slots, 0);
}

int ConfigRegistry::assign(int slot, const CfgConst& k, bool* build) {
    *build = false;
    const int old = slot_var_[slot];
    if (std::memcmp(&vars_[old].k, &k, sizeof(k)) == 0) return old;
    --vars_[old].refs;
    // a variant with these constants, used or not (an unused one still holds intact device data)
    int id = -1;
    for (int i = 0; i < (int)vars_.size() && id < 0; ++i)
        if (std::memcmp(&vars_[i].k, &k, sizeof(k)) == 0) id = i;
    if (id < 0) {
        for (int i = 0; i < (int)vars_.size() && id < 0; ++i)
            if (vars_[i].refs == 0) id = i;
        if (id < 0) {
            id = (int)vars_.size();
            vars_.push_back(Variant{});
        }
        vars_[id].k = k;
        *build = true;
    }
    ++vars_[id].refs;
    slot_var_[slot] = id;
    return id;
}

int ConfigRegistry::live() const {
    int n = 0;
    for (const Variant& v : vars_) n += v.refs > 0;
    return n;
}

// grid_map::GridMap::move (getIndexShiftFromPositionShift / getPositionShiftFromIndexShift):
// whole-cell shift, rounded half away from zero; the map position advances by the aligned
// shift.  Returns the buffer index shift: new(r, c) = old(r + shift_i, c + shift_j).
void move_map(double res, double& px, double& py, double nx, double ny, int& shift_i, int& shift_j) {
    const double tx = (nx - px) / res, ty = (ny - py) / res;
    const int cx = (int)(tx + 0.5 * (tx > 0 ? 1 : -1));
    const int cy = (int)(ty + 0.5 * (ty > 0 ? 1 : -1));
    shift_i = -cx;
    shift_j = -cy;
    px += (double)cx * res;
    py += (double)cy * res;
}

// Wavefront schedule of GroundSegmentation::spiral_ground_interpolation (:398-441).
// Every visit reads the 3x3 neighbourhood of G and C and writes its own cell (:453-464).
// level(v) = 1 + max(level of the last writer of any cell it reads, level of any earlier
// reader of the cell it writes); visits of one level are mutually independent, so running
// the levels in order reproduces the sequential sweep exactly.
void build_spiral_schedule(int n, std::vector<int>& level_start, std::vector<uint32_t>& visits) {
    const int c = n / 2 - 1;
    std::vector<int> last_write((size_t)n * n, -1), last_read((size_t)n * n, -1);
    std::vector<uint32_t> seq;
    std::vector<int> lvl;
    auto visit = [&](int x, int y) {
        int l = 0;
        for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx) l = std::max(l, last_write[(x + dx) + (size_t)(y + dy) * n] + 1);
        l = std::max(l, last_read[x + (size_t)y * n] + 1);
        for (int dy = -1; dy <= 1; ++dy)
            for (int dx = -1; dx <= 1; ++dx) {
                int& r = last_read[(x + dx) + (size_t)(y + dy) * n];
                r = std::max(r, l);
            }
        last_write[x + (size_t)y * n] = l;
        seq.push_back((uint32_t)x | ((uint32_t)y << 16));
        lvl.push_back(l);
    };
    for (int p = c - 1; p >= 1; --p) {
        const int side = (c - p) * 2;
        const int q = p + side;
        for (int pos = p; pos < q; ++pos) visit(p, pos);       // side 0: x fixed
        for (int pos = p; pos < q; ++pos) visit(pos, p);       // side 1: y fixed
        for (int pos = q; pos >= p; --pos) visit(q, pos);      // far sides, descending
        for (int pos = q; pos >= p; --pos) visit(pos, q);
    }
    int levels = 0;
    for (int l : lvl) levels = std::max(levels, l + 1);
    level_start.assign((size_t)levels + 1, 0);
    for (int l : lvl) ++level_start[(size_t)l + 1];
    for (int l = 0; l < levels; ++l) level_start[(size_t)l + 1] += level_start[l];
    visits.resize(seq.size());
    std::vector<int> cursor(level_start.begin(), level_start.end() - 1);
    for (size_t v = 0; v < seq.size(); ++v) visits[(size_t)cursor[lvl[v]]++] = seq[v];
}

// Schedule records for the pipelined spiral kernel (k_spiral_pipe): per visit
//   w0 = x | y << 16
//   w1, w2 = up to four "recent" entries (16 bit each): bits 14..15 = how many levels earlier
//            the neighbour was written (1..3, 0 = unused entry), bits 10..13 neighbour index q
//            (block(q % 3, q / 3) of the 3x3 neighbourhood), bits 0..9 the slot (index inside
//            its level) of the visit that wrote it
//   w3 = bit 0: the cell lies beyond minDistSquared (confidence decays, :463-464)
//        bit 1: second visit of this cell (ring corners are visited twice, :421-438)
// The kernel prefetches a visit's 3x3 neighbourhood `dist` levels ahead; a neighbour written
// less than `dist` levels before the visit cannot come from that prefetch and is delivered
// through shared memory instead.  Returns false if a visit needs more than four such recents
// or a level has more than 1024 visits (the caller then uses the plain k_spiral).
bool build_spiral_records(int n, double res_sq, const std::vector<int>& level_start, const std::vector<uint32_t>& visits,
                          int dist, std::vector<uint32_t>& recs, int& max_recent) {
    const int c = n / 2 - 1;
    const size_t nv = visits.size();
    if (dist < 1 || dist > 3) return false;
    // level and slot of every visit, looked up by (level-sorted) position
    std::vector<int> level_of(nv), slot_of(nv);
    for (size_t l = 0; l + 1 < level_start.size(); ++l) {
        if (level_start[l + 1] - level_start[l] > 1024) return false;
        for (int t = level_start[l]; t < level_start[l + 1]; ++t) {
            level_of[t] = (int)l;
            slot_of[t] = t - level_start[l];
        }
    }
    // Replay the sequential order to know, for each visit, the last writer of every neighbour.
    // Sequential order != level-sorted order, so map (cell, occurrence) -> sorted position.
    std::vector<std::vector<int>> pos_of_cell((size_t)n * n);
    for (size_t t = 0; t < nv; ++t) {
        const int x = visits[t] & 0xffff, y = visits[t] >> 16;
        pos_of_cell[x + (size_t)y * n].push_back((int)t);  // level order == visit order for one cell (WAW)
    }
    std::vector<int> seen((size_t)n * n, 0);      // how many visits of the cell happened so far
    std::vector<int> last_writer((size_t)n * n, -1);  // sorted position of the cell's last writer
    recs.assign(nv * 4, 0u);
    max_recent = 0;
    bool ok = true;
    auto visit = [&](int x, int y) {
        const size_t cell = x + (size_t)y * n;
        const int t = pos_of_cell[cell][seen[cell]];
        const int lvl = level_of[t];
        uint32_t r[4] = {0, 0, 0, 0};
        int nr = 0;
        for (int q = 0; q < 9; ++q) {
            const size_t nb = (size_t)(x - 1 + q % 3) + (size_t)(y - 1 + q / 3) * n;
            const int w = last_writer[nb];
            if (w >= 0 && level_of[w] < lvl && level_of[w] >= lvl - dist) {
                // bits 14..15: how many levels earlier the neighbour was written (1 .. dist <= 3); 0 = unused entry
                if (nr < 4) r[nr] = ((uint32_t)(lvl - level_of[w]) << 14) | ((uint32_t)q << 10) | (uint32_t)slot_of[w];
                ++nr;
            } else if (w >= 0 && level_of[w] >= lvl) {
                ok = false;  // would contradict the levelisation
            }
        }
        if (nr > 4) ok = false;
        max_recent = std::max(max_recent, nr);
        const float fx = (float)x - (float)c, fy = (float)y - (float)c;
        const bool far = ((double)fx * (double)fx + (double)fy * (double)fy) * res_sq > 12.0;
        recs[4 * (size_t)t + 0] = (uint32_t)x | ((uint32_t)y << 16);
        recs[4 * (size_t)t + 1] = r[0] | (r[1] << 16);
        recs[4 * (size_t)t + 2] = r[2] | (r[3] << 16);
        recs[4 * (size_t)t + 3] = (far ? 1u : 0u) | (seen[cell] ? 2u : 0u);  // bit 1: second visit of a ring corner
        last_writer[cell] = t;
        ++seen[cell];
    };
    for (int p = c - 1; p >= 1; --p) {
        const int side = (c - p) * 2;
        const int q = p + side;
        for (int pos = p; pos < q; ++pos) visit(p, pos);
        for (int pos = p; pos < q; ++pos) visit(pos, p);
        for (int pos = q; pos >= p; --pos) visit(q, pos);
        for (int pos = q; pos >= p; --pos) visit(pos, q);
    }
    return ok;
}

// ---- skewed-layout tables for k_spiral_skew ----------------------------------------------
// The sweep consists of "lanes": ring k (p = c-1-k, L = 2(k+1), q = p+L) has four sides that the
// sequential order walks cell by cell (side 0: (p, p+j), side 1: (p+j, p), side 2: (q, q-j),
// side 3: (q-j, q)).  In the levelised schedule a lane advances one cell per level for almost all
// of its length, and ring k+1 trails ring k by three levels.  Storing the value visited by lane
// (s, k) at level l in slot (s, l, k) therefore makes the 3x3 neighbourhood of a visit a FIXED
// offset pattern in (level, ring) space, and 32 consecutive rings of one side (a warp) read 32
// consecutive slots: every load of the hot loop is coalesced.  Visits that do not follow the
// pattern (first / last cells of a lane, ring corners with two homes) are "irregular": they carry
// explicit slot indices and are executed by a dedicated warp.
void build_spiral_skew(int n, const std::vector<int>& level_start, const std::vector<uint32_t>& visits, SkewTables& t) {
    t = SkewTables();
    t.n = n;
    const int c = n / 2 - 1;
    const int K = c - 1;
    t.K = K;
    t.levels = (int)level_start.size() - 1;
    if (K < 2) return;
    t.KP = ((K + 2 + 31) / 32) * 32;
    if (4 * t.KP > 4095) return;  // lane ids travel in 12 bits
    const size_t nv = visits.size();
    // level of the i-th visit of every cell (level order == visit order per cell)
    std::vector<std::vector<int>> cell_levels((size_t)n * n);
    for (int l = 0; l < t.levels; ++l)
        for (int v = level_start[l]; v < level_start[l + 1]; ++v) {
            const int x = visits[v] & 0xffff, y = visits[v] >> 16;
            cell_levels[x + (size_t)y * n].push_back(l);
        }
    struct Visit {
        int s, k, j, x, y, level;
    };
    std::vector<Visit> seq;
    seq.reserve(nv);
    std::vector<int> seen((size_t)n * n, 0);
    int max_level = 0;
    auto push = [&](int s, int k, int j, int x, int y) {
        const size_t cell = x + (size_t)y * n;
        const int l = cell_levels[cell][seen[cell]++];
        seq.push_back({s, k, j, x, y, l});
        max_level = std::max(max_level, l);
    };
    for (int k = 0; k < K; ++k) {
        const int p = c - 1 - k, L = 2 * (k + 1), q = p + L;
        for (int j = 0; j < L; ++j) push(0, k, j, p, p + j);
        for (int j = 0; j < L; ++j) push(1, k, j, p + j, p);
        for (int j = 0; j <= L; ++j) push(2, k, j, q, q - j);
        for (int j = 0; j <= L; ++j) push(3, k, j, q - j, q);
    }
    if (seq.size() != nv) return;
    // start level of every lane must be 3k + off[s] (checked), used to place the never-visited cells
    int off[4] = {0, 0, 0, 0};
    const int k_ref = K / 2;  // the innermost rings start irregularly; take the offsets from a middle ring
    for (const Visit& v : seq)
        if (v.k == k_ref && v.j == 0) off[v.s] = v.level - 3 * k_ref;
    for (const Visit& v : seq)
        if (v.k >= 4 && v.j == 0 && v.level != 3 * v.k + off[v.s]) return;
    const int LK = 2 * (K + 1);
    t.rows = std::max(max_level, 3 * K + off[3] + LK + 1) + t.row0 + 8;
    t.lanes = 4 * t.KP;
    t.slots = (size_t)4 * t.rows * t.KP;
    auto slot = [&](int s, int k, int level) { return (int)(((size_t)s * t.rows + level + t.row0) * t.KP + (k + 1)); };

    // homes of every cell: slots of its visits; never-visited cells that are read as neighbours
    // (centre, outermost border ring) sit where a virtual lane would visit them
    t.cell_home.assign((size_t)n * n * 4, -1);
    auto add_home = [&](int x, int y, int sl) {
        int* h = &t.cell_home[((size_t)x + (size_t)y * n) * 4];
        for (int i = 0; i < 4; ++i)
            if (h[i] < 0) {
                h[i] = sl;
                return;
            }
    };
    for (const Visit& v : seq) add_home(v.x, v.y, slot(v.s, v.k, v.level));
    {
        const int p = 0, k = K, q = p + LK;  // virtual ring K: the border the outermost ring reads
        if (q < n) {
            for (int j = 0; j < LK; ++j) add_home(p, p + j, slot(0, k, 3 * k + off[0] + j));
            for (int j = 1; j < LK; ++j) add_home(p + j, p, slot(1, k, 3 * k + off[1] + j));  // (p, p) already has its side-0 home
            for (int j = 0; j <= LK; ++j) add_home(q, q - j, slot(2, k, 3 * k + off[2] + j));
            for (int j = 1; j <= LK; ++j)
                if (!(q - j == p)) add_home(q - j, q, slot(3, k, 3 * k + off[3] + j));         // (p, q) keeps a single home below
            add_home(p, q, slot(3, k, 3 * k + off[3] + LK));
        }
        for (int s = 0; s < 4; ++s) add_home(c, c, slot(s, -1, -3 + off[s]));  // centre: virtual ring -1
    }
    auto homes = [&](int x, int y) { return &t.cell_home[((size_t)x + (size_t)y * n) * 4]; };
    // the cells whose homes the closed form does not give (k_detect stores those from cell_home)
    std::memcpy(t.off, off, sizeof(off));
    t.home_words = (n + 31) / 32;
    t.home_irr.assign((size_t)n * t.home_words, 0u);
    for (int y = 0; y < n; ++y)
        for (int x = 0; x < n; ++x) {
            const int* h = homes(x, y);
            if (h[0] != skew_regular_home(n, K, t.KP, t.rows, t.row0, t.off, x, y) || h[1] >= 0)
                t.home_irr[(size_t)y * t.home_words + x / 32] |= 1u << (x % 32);
        }

    // neighbour slot candidates + offset statistics -> the regular pattern of each side
    std::vector<std::vector<std::pair<int, int>>> stat(36);  // (offset, count), small
    auto bump = [&](int idx, int o) {
        for (auto& e : stat[idx])
            if (e.first == o) {
                ++e.second;
                return;
            }
        stat[idx].push_back({o, 1});
    };
    for (const Visit& v : seq) {
        if (v.j < 3 || v.k < 4) continue;  // statistics from lane interiors only
        const int own = slot(v.s, v.k, v.level);
        for (int q = 0; q < 9; ++q) {
            const int* h = homes(v.x - 1 + q % 3, v.y - 1 + q / 3);
            for (int i = 0; i < 4 && h[i] >= 0; ++i) bump(v.s * 9 + q, h[i] - own);
        }
    }
    for (int i = 0; i < 36; ++i) {
        int best = 0, cnt = -1;
        for (auto& e : stat[i])
            if (e.second > cnt) {
                cnt = e.second;
                best = e.first;
            }
        if (cnt < 0) return;
        t.pattern[i] = best;
    }

    // classify visits; irregular ones get explicit records
    std::vector<int> last_level((size_t)n * n, -1000000), last_lane((size_t)n * n, -1);
    t.lane_begin.assign(t.lanes, 0);
    t.lane_end.assign(t.lanes, 0);
    t.lane_cell0.assign(t.lanes, 0);
    std::vector<int> reg_first(t.lanes, -1), reg_last(t.lanes, -1), reg_count(t.lanes, 0);
    struct Irr {
        int level;
        uint32_t w[16];
    };
    std::vector<Irr> irr;
    for (const Visit& v : seq) {
        const int lane = v.s * t.KP + (v.k + 1);
        const int own = slot(v.s, v.k, v.level);
        const size_t cell = v.x + (size_t)v.y * n;
        int nb[9];
        bool regular = true;
        uint32_t rec[4] = {0xffffu, 0xffffu, 0xffffu, 0xffffu};  // (q << 12) | producer lane, 0xffff = unused
        int nrec = 0;
        for (int q = 0; q < 9; ++q) {
            const int cx = v.x - 1 + q % 3, cy = v.y - 1 + q / 3;
            const int* h = homes(cx, cy);
            if (h[0] < 0) return;  // a neighbour without a home: geometry not covered
            const int want = own + t.pattern[v.s * 9 + q];
            bool match = false;
            for (int i = 0; i < 4 && h[i] >= 0; ++i) match |= (h[i] == want);
            nb[q] = match ? want : h[0];
            if (!match) regular = false;
            const size_t ncell = cx + (size_t)cy * n;
            const int back = v.level - last_level[ncell];
            if (back < 1) return;  // contradicts the levelisation
            if (back == 1) {        // written one level ago: travels through shared memory
                if (!(q == t.prev_q[v.s] && last_lane[ncell] == lane)) regular = false;
                if (nrec < 4) rec[nrec] = ((uint32_t)q << 12) | (uint32_t)last_lane[ncell];
                ++nrec;
            }
        }
        if (nrec > 4) return;
        if (nrec != 1) regular = false;  // a lane thread always takes its previous cell from the exchange buffer
        const int* hown = homes(v.x, v.y);
        int mirror = -1;
        if (hown[1] >= 0) {
            regular = false;  // a ring corner: both homes are kept identical
            mirror = (hown[0] == own) ? hown[1] : hown[0];
            if (hown[2] >= 0) return;
        }
        if (regular) {
            ++t.n_regular;
            if (reg_first[lane] < 0) {
                reg_first[lane] = v.level;
                t.lane_cell0[lane] = (int)cell;
            }
            if (reg_last[lane] >= 0 && v.level != reg_last[lane] + 1) return;  // the regular run must be contiguous in levels
            reg_last[lane] = v.level;
            ++reg_count[lane];
        } else {
            ++t.n_irregular;
            Irr r;
            r.level = v.level;
            std::memset(r.w, 0, sizeof(r.w));
            r.w[0] = (uint32_t)own;
            for (int q = 0; q < 9; ++q) r.w[1 + q] = (uint32_t)nb[q];
            r.w[10] = rec[0] | (rec[1] << 16);
            r.w[11] = rec[2] | (rec[3] << 16);
            r.w[12] = (uint32_t)mirror;
            r.w[13] = (uint32_t)lane;
            r.w[14] = (uint32_t)cell;
            irr.push_back(r);
        }
        last_level[cell] = v.level;
        last_lane[cell] = lane;
    }
    for (int l = 0; l < t.lanes; ++l)
        if (reg_first[l] >= 0) {
            t.lane_begin[l] = reg_first[l];
            t.lane_end[l] = reg_last[l] + 1;
            if (t.lane_end[l] - t.lane_begin[l] != reg_count[l]) return;
        }
    // CSR of the irregular visits by level
    t.irr_level_start.assign((size_t)t.levels + 1, 0);
    for (const Irr& r : irr) ++t.irr_level_start[(size_t)r.level + 1];
    for (int l = 0; l < t.levels; ++l) {
        t.max_irr_per_level = std::max(t.max_irr_per_level, t.irr_level_start[(size_t)l + 1]);
        t.irr_level_start[(size_t)l + 1] += t.irr_level_start[l];
    }
    if (t.max_irr_per_level > 32) return;
    t.irr_recs.assign(irr.size() * 16, 0u);
    std::vector<int> cur(t.irr_level_start.begin(), t.irr_level_start.end() - 1);
    for (const Irr& r : irr) std::memcpy(&t.irr_recs[(size_t)cur[r.level]++ * 16], r.w, sizeof(r.w));
    t.ok = true;
}

// The path choice, in order of preference:
//   1. skew, when build_spiral_skew covers the geometry and one CTA holds the layout.  One lane thread per lane when that
//      fits (measured fastest, for single scans and batches alike, DESIGN.md section 3.3); otherwise lane threads are
//      time-shared: the smallest M (multiple of 32) such that ring k + M of a side starts (prefetch window included)
//      only after ring k has finished.
//   2. pipe, when every level has at most 1024 visits and build_spiral_records succeeds.
//   3. plain k_spiral.
void plan_spiral(int n, double res_sq, SpiralPlan& p) {
    p = SpiralPlan();
    build_spiral_schedule(n, p.level_start, p.visits);
    for (size_t l = 0; l + 1 < p.level_start.size(); ++l) p.max_per_level = std::max(p.max_per_level, p.level_start[l + 1] - p.level_start[l]);

    SkewTables& sk = p.skew;
    build_spiral_skew(n, p.level_start, p.visits, sk);
    if (sk.ok) {
        int M = sk.KP;
        if (4 * sk.KP + SKEW_IRR_THREADS > 1024) {
            const int kGap = 2 * 8 + 4;  // 2 * PF_FAR of k_spiral_skew + slack
            for (M = 32; M < sk.KP; M += 32) {
                bool fits = true;
                for (int sd = 0; sd < 4 && fits; ++sd)
                    for (int c0 = 0; c0 + M < sk.KP && fits; ++c0) {
                        const int a = sd * sk.KP + c0, b2 = a + M;
                        if (sk.lane_begin[a] < sk.lane_end[a] && sk.lane_begin[b2] < sk.lane_end[b2] && sk.lane_end[a] + kGap > sk.lane_begin[b2])
                            fits = false;
                    }
                if (fits) break;
            }
            M = std::min(M, sk.KP);
        }
        // one CTA: lane threads + the two irregular warps (one thread per (visit, neighbour))
        if (4 * M + SKEW_IRR_THREADS <= 1024 && sk.max_irr_per_level * 9 <= SKEW_IRR_THREADS) {
            p.kind = SPIRAL_SKEW;
            p.M = M;
            p.phases = (sk.KP + M - 1) / M;
            p.threads = 4 * M + SKEW_IRR_THREADS;
            // [phase][side * M + m] tables of the lane threads
            const size_t cols = (size_t)p.phases * 4 * M;
            p.ph_begin.assign(cols, 0);
            p.ph_end.assign(cols, 0);
            p.ph_cell0.assign(cols, 0);
            for (int ph = 0; ph < p.phases; ++ph)
                for (int sd = 0; sd < 4; ++sd)
                    for (int m = 0; m < M; ++m) {
                        const int col = ph * M + m;
                        if (col >= sk.KP) continue;
                        const size_t dst = ((size_t)ph * 4 + sd) * M + m;
                        p.ph_begin[dst] = sk.lane_begin[sd * sk.KP + col];
                        p.ph_end[dst] = sk.lane_end[sd * sk.KP + col];
                        p.ph_cell0[dst] = sk.lane_cell0[sd * sk.KP + col];
                    }
            // re-layout of the irregular records: one dense block per level (see SkewView)
            p.irr_max = std::max(1, sk.max_irr_per_level);
            const int irr_words = ((p.irr_max * 22 + 3) / 4) * 4;
            p.irr_chunks = irr_words / 4;
            p.irr_blocks.assign((size_t)(sk.levels + 4) * irr_words, 0xffffffffu);
            for (int l = 0; l < sk.levels; ++l)
                for (int r = sk.irr_level_start[l]; r < sk.irr_level_start[l + 1]; ++r) {
                    const uint32_t* w = &sk.irr_recs[(size_t)r * 16];
                    const int vv = r - sk.irr_level_start[l];
                    uint32_t* blk = &p.irr_blocks[(size_t)l * irr_words];
                    for (int q = 0; q < 9; ++q) {
                        blk[(vv * 9 + q) * 2] = w[1 + q];
                        blk[(vv * 9 + q) * 2 + 1] = 0xffffffffu;
                    }
                    const uint32_t ents[4] = {w[10] & 0xffffu, w[10] >> 16, w[11] & 0xffffu, w[11] >> 16};
                    for (uint32_t e : ents)
                        if (e != 0xffffu) blk[(vv * 9 + (e >> 12)) * 2 + 1] = e & 4095u;
                    uint32_t* hd = blk + p.irr_max * 18 + vv * 4;
                    hd[0] = w[0];
                    hd[1] = w[12];
                    hd[2] = w[13];
                    hd[3] = w[14];
                }
            return;
        }
    }
    int max_recent = 0;
    if (p.max_per_level <= 1024 && build_spiral_records(n, res_sq, p.level_start, p.visits, SPIRAL_PIPE_DIST, p.recs, max_recent)) {
        p.kind = SPIRAL_PIPE;
        p.threads = p.max_per_level <= 512 ? 512 : 1024;
        return;
    }
    p.threads = SPIRAL_THREADS;
}

// ---- host-side cloud packing (gg_filter_cloud_batch) -------------------------------------
// PointXYZIR records (32 B, 14 useful) -> x | y | z (float[n_pad]) | ring (u16[n_pad]) with
// n_pad = n rounded up to 8, written with streaming stores into pinned staging memory.
// [i0, i1) is a chunk: i0 a multiple of 8, i1 == n for the last chunk (which also zero-fills
// the padding).  AVX2 variant selected at run time.
static void pack_tail(const gg_point* src, size_t n, size_t n_pad, float* x, float* y, float* z, uint16_t* r, size_t i, size_t i1) {
    for (; i < i1 && i < n; ++i) {
        x[i] = src[i].x;
        y[i] = src[i].y;
        z[i] = src[i].z;
        r[i] = src[i].ring;
    }
    if (i1 >= n)
        for (size_t t = n; t < n_pad; ++t) {
            x[t] = y[t] = z[t] = 0.f;
            r[t] = 0;
        }
}

static void pack_sse2(const gg_point* src, size_t n, unsigned char* dst, size_t i0, size_t i1) {
    const size_t n_pad = (n + 7) & ~(size_t)7;
    float* x = reinterpret_cast<float*>(dst);
    float* y = x + n_pad;
    float* z = y + n_pad;
    uint16_t* r = reinterpret_cast<uint16_t*>(z + n_pad);
    size_t i = i0;
    const size_t vec_end = i0 + ((std::min(i1, n) - i0) & ~(size_t)7);
    for (; i < vec_end; i += 8) {
        alignas(16) uint16_t rr[8];
        for (int h = 0; h < 2; ++h) {
            const gg_point* p = src + i + 4 * h;
            __m128 a = _mm_loadu_ps(&p[0].x), b = _mm_loadu_ps(&p[1].x), c = _mm_loadu_ps(&p[2].x), d = _mm_loadu_ps(&p[3].x);
            _MM_TRANSPOSE4_PS(a, b, c, d);  // a = x0..x3, b = y0..y3, c = z0..z3
            _mm_stream_ps(x + i + 4 * h, a);
            _mm_stream_ps(y + i + 4 * h, b);
            _mm_stream_ps(z + i + 4 * h, c);
            for (int q = 0; q < 4; ++q) rr[4 * h + q] = p[q].ring;
        }
        _mm_stream_si128(reinterpret_cast<__m128i*>(r + i), _mm_load_si128(reinterpret_cast<const __m128i*>(rr)));
    }
    pack_tail(src, n, n_pad, x, y, z, r, i, i1);
    _mm_sfence();
}

// 32 records (1 KB) per iteration: every destination cache line (2 of x, y and z each, 1 of rings) is
// written completely by back-to-back streaming stores, so each write-combining buffer drains as one full
// line.  The rings come out of the upper record halves by the same in-lane transpose as the coordinates.
__attribute__((target("avx2"))) static inline void pack8_avx2(const gg_point* p, float* x, float* y, float* z, __m256i& ring_dwords) {
    // lane 0: records 0..3, lane 1: records 4..7; transpose 4x4 inside each 128-bit lane
    const __m256 a = _mm256_loadu2_m128(&p[4].x, &p[0].x), b = _mm256_loadu2_m128(&p[5].x, &p[1].x);
    const __m256 c = _mm256_loadu2_m128(&p[6].x, &p[2].x), d = _mm256_loadu2_m128(&p[7].x, &p[3].x);
    const __m256 t0 = _mm256_unpacklo_ps(a, b), t1 = _mm256_unpackhi_ps(a, b);
    const __m256 t2 = _mm256_unpacklo_ps(c, d), t3 = _mm256_unpackhi_ps(c, d);
    const __m256 vx = _mm256_shuffle_ps(t0, t2, 0x44), vy = _mm256_shuffle_ps(t0, t2, 0xEE), vz = _mm256_shuffle_ps(t1, t3, 0x44);  // x0..x3 | x4..x7
    _mm256_stream_ps(x, vx);
    _mm256_stream_ps(y, vy);
    _mm256_stream_ps(z, vz);
    // upper halves: intensity | ring (u16) + 2 padding bytes | padding | padding
    const __m256 e = _mm256_loadu2_m128(&p[4].intensity, &p[0].intensity), f = _mm256_loadu2_m128(&p[5].intensity, &p[1].intensity);
    const __m256 g = _mm256_loadu2_m128(&p[6].intensity, &p[2].intensity), h = _mm256_loadu2_m128(&p[7].intensity, &p[3].intensity);
    const __m256 u0 = _mm256_unpacklo_ps(e, f), u2 = _mm256_unpacklo_ps(g, h);
    ring_dwords = _mm256_and_si256(_mm256_castps_si256(_mm256_shuffle_ps(u0, u2, 0xEE)), _mm256_set1_epi32(0xffff));
}

// records to prefetch ahead of the 32 being packed: 256 records are 8 KB, which lands in L1 before they are read
constexpr int kPackPrefetchRecords = 256;

__attribute__((target("avx2"))) static void pack_avx2(const gg_point* src, size_t n, unsigned char* dst, size_t i0, size_t i1) {
    const size_t n_pad = (n + 7) & ~(size_t)7;
    float* x = reinterpret_cast<float*>(dst);
    float* y = x + n_pad;
    float* z = y + n_pad;
    uint16_t* r = reinterpret_cast<uint16_t*>(z + n_pad);
    size_t i = i0;
    const size_t stop = std::min(i1, n);
    const size_t end32 = i0 + ((stop - i0) & ~(size_t)31), end8 = i0 + ((stop - i0) & ~(size_t)7);
    for (; i < end32; i += 32) {
        const gg_point* p = src + i;
        // 1 KB of records per iteration, prefetched into L1 (prefetcht0) 8 KB ahead
        const char* pf = reinterpret_cast<const char*>(p + kPackPrefetchRecords);
        for (int l = 0; l < 16; ++l) _mm_prefetch(pf + 64 * l, _MM_HINT_T0);
        __m256i r0, r1, r2, r3;
        // coordinates line by line: 16 records fill one 64-byte line of x, y and z each
        pack8_avx2(p, x + i, y + i, z + i, r0);
        pack8_avx2(p + 8, x + i + 8, y + i + 8, z + i + 8, r1);
        pack8_avx2(p + 16, x + i + 16, y + i + 16, z + i + 16, r2);
        pack8_avx2(p + 24, x + i + 24, y + i + 24, z + i + 24, r3);
        // packus interleaves the 128-bit lanes of its operands: restore record order with a 64-bit permute
        const __m256i w0 = _mm256_permute4x64_epi64(_mm256_packus_epi32(r0, r1), 0xD8), w1 = _mm256_permute4x64_epi64(_mm256_packus_epi32(r2, r3), 0xD8);
        _mm256_stream_si256(reinterpret_cast<__m256i*>(r + i), w0);
        _mm256_stream_si256(reinterpret_cast<__m256i*>(r + i + 16), w1);
    }
    for (; i < end8; i += 8) {
        __m256i r0;
        pack8_avx2(src + i, x + i, y + i, z + i, r0);
        const __m256i w = _mm256_permute4x64_epi64(_mm256_packus_epi32(r0, r0), 0xD8);
        _mm_store_si128(reinterpret_cast<__m128i*>(r + i), _mm256_castsi256_si128(w));
    }
    pack_tail(src, n, n_pad, x, y, z, r, i, i1);
    _mm_sfence();
}

void pack_cloud_range(const gg_point* src, size_t n, unsigned char* dst, size_t i0, size_t i1) {
    static const bool have_avx2 = __builtin_cpu_supports("avx2");
    if (have_avx2 && (reinterpret_cast<uintptr_t>(dst) & 31) == 0)
        pack_avx2(src, n, dst, i0, i1);
    else
        pack_sse2(src, n, dst, i0, i1);
}

// CPUs this process may actually use: affinity mask capped by the cgroup CPU quota
int usable_cpus() {
    int n = (int)std::thread::hardware_concurrency();
#ifdef __linux__
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof(set), &set) == 0) n = std::min(n, CPU_COUNT(&set));
    if (FILE* f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char quota[32];
        long period = 0;
        if (std::fscanf(f, "%31s %ld", quota, &period) == 2 && period > 0 && quota[0] != 'm') n = std::min(n, (int)std::max(1L, std::atol(quota) / period));
        std::fclose(f);
    } else if (FILE* f1 = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
        long q = -1, per = 100000;
        if (std::fscanf(f1, "%ld", &q) != 1) q = -1;
        std::fclose(f1);
        if (FILE* f2 = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
            if (std::fscanf(f2, "%ld", &per) != 1) per = 100000;
            std::fclose(f2);
        }
        if (q > 0 && per > 0) n = std::min(n, (int)std::max(1L, q / per));
    }
#endif
    return std::max(1, n);
}

}  // namespace gg

extern "C" {

int gg_host_cells_per_side(double dimension_m, float resolution) { return gg::cells_per_side(dimension_m, resolution); }

int gg_host_expected_points(double dimension_m, float resolution, float* dst) {
    std::vector<float> t;
    const int n = gg::cells_per_side(dimension_m, resolution);
    gg::build_expected_points(n, t);
    std::memcpy(dst, t.data(), t.size() * sizeof(float));
    return n;
}

int gg_host_spiral_schedule(int n, int* level_start, int level_cap, uint32_t* visits, int visit_cap, int* n_levels, int* n_visits) {
    std::vector<int> ls;
    std::vector<uint32_t> vs;
    gg::build_spiral_schedule(n, ls, vs);
    *n_levels = (int)ls.size() - 1;
    *n_visits = (int)vs.size();
    if (level_start && level_cap >= (int)ls.size()) std::memcpy(level_start, ls.data(), ls.size() * sizeof(int));
    if (visits && visit_cap >= (int)vs.size()) std::memcpy(visits, vs.data(), vs.size() * sizeof(uint32_t));
    return 0;
}

// records of the pipelined spiral kernel: 4 uint32 per visit (see build_spiral_records)
int gg_host_spiral_records(int n, float resolution, int dist, uint32_t* recs, int rec_cap_words, int* max_recent) {
    std::vector<int> ls;
    std::vector<uint32_t> vs, rc;
    gg::build_spiral_schedule(n, ls, vs);
    int mr = 0;
    const bool ok = gg::build_spiral_records(n, (double)resolution * (double)resolution, ls, vs, dist, rc, mr);
    if (max_recent) *max_recent = mr;
    if (recs && rec_cap_words >= (int)rc.size()) std::memcpy(recs, rc.data(), rc.size() * sizeof(uint32_t));
    return ok ? 1 : 0;
}

// out[4]: the spiral path of a map (see plan_spiral): kind (gg::SpiralKind), CTA threads, M, phases
int gg_host_spiral_plan(int n, float resolution, int* out) {
    gg::SpiralPlan p;
    gg::plan_spiral(n, (double)resolution * (double)resolution, p);
    const int v[4] = {(int)p.kind, p.threads, p.M, p.phases};
    std::memcpy(out, v, sizeof(v));
    return 0;
}

// header: ok, K, KP, rows, levels, row0, lanes, n_irregular, max_irr_per_level, n_regular
int gg_host_spiral_skew(int n, int* header, int* pattern, int* lane_begin, int* lane_end, int* cell_home, int* irr_level_start,
                        uint32_t* irr_recs, int irr_cap_words) {
    std::vector<int> ls;
    std::vector<uint32_t> vs;
    gg::build_spiral_schedule(n, ls, vs);
    gg::SkewTables t;
    gg::build_spiral_skew(n, ls, vs, t);
    const int h[10] = {t.ok ? 1 : 0, t.K, t.KP, t.rows, t.levels, t.row0, t.lanes, (int)t.n_irregular, t.max_irr_per_level, (int)t.n_regular};
    std::memcpy(header, h, sizeof(h));
    if (!t.ok) return 0;
    if (pattern) std::memcpy(pattern, t.pattern, sizeof(t.pattern));
    if (lane_begin) std::memcpy(lane_begin, t.lane_begin.data(), t.lane_begin.size() * sizeof(int));
    if (lane_end) std::memcpy(lane_end, t.lane_end.data(), t.lane_end.size() * sizeof(int));
    if (cell_home) std::memcpy(cell_home, t.cell_home.data(), t.cell_home.size() * sizeof(int));
    if (irr_level_start) std::memcpy(irr_level_start, t.irr_level_start.data(), t.irr_level_start.size() * sizeof(int));
    if (irr_recs && irr_cap_words >= (int)t.irr_recs.size()) std::memcpy(irr_recs, t.irr_recs.data(), t.irr_recs.size() * sizeof(uint32_t));
    return 1;
}

int gg_host_skew_homes(int n, int* homes, int* n_table) {
    std::vector<int> ls;
    std::vector<uint32_t> vs;
    gg::build_spiral_schedule(n, ls, vs);
    gg::SkewTables t;
    gg::build_spiral_skew(n, ls, vs, t);
    if (!t.ok) return 0;
    gg::SkewView w;
    std::memset(&w, 0, sizeof(w));
    w.cell_home = t.cell_home.data();
    w.home_irr = t.home_irr.data();
    w.home_words = t.home_words;
    w.K = t.K;
    w.KP = t.KP;
    w.rows = t.rows;
    w.row0 = t.row0;
    std::memcpy(w.off, t.off, sizeof(t.off));
    int table = 0;
    for (int y = 0; y < n; ++y)
        for (int x = 0; x < n; ++x) {
            const int4 h = gg::skew_home(w, n, x, y);
            int* o = homes + ((size_t)x + (size_t)y * n) * 4;
            o[0] = h.x;
            o[1] = h.y;
            o[2] = h.z;
            o[3] = h.w;
            table += (t.home_irr[(size_t)y * t.home_words + x / 32] >> (x % 32)) & 1u;
        }
    *n_table = table;
    return 1;
}

// the confidence decay of every spiral path (gg_internal.h:decay_confidence) for the configuration cfg, on the host
int gg_host_decay_confidence(const gg_config* cfg, const float* occ, size_t n, float* out) {
    gg::CfgConst k;
    gg::derive_config(*cfg, k);
    for (size_t i = 0; i < n; ++i) out[i] = gg::decay_confidence(k, occ[i]);
    return 0;
}

// the confidence a visit of k_spiral_skew leaves: its SD entry d, or the visited cell's own occ where d is SKEW_NEAR
int gg_host_skew_visit_confidence(const float* d, const float* occ, size_t n, float* out) {
    for (size_t i = 0; i < n; ++i) out[i] = gg::skew_decays(d[i]) ? d[i] : occ[i];
    return 0;
}

// The outlier ray-march of k_rasterize from step `from` on (gg_internal.h:outlier_walk), for the ray from `origin` to
// `point` (x, y, z) over the prior G / C of an N x N map at pos_xy: 1 an occluding cell is found, 0 none, -1 the ray does
// not march (vz is not below -0.01f).  The direction is k_rasterize's (:250-257).
int gg_host_outlier_walk(double dimension_m, float resolution, const double* pos_xy, const float* G, const float* C, double thr, double tol,
                         const float* origin, const float* point, long long from) {
    gg::Const k;
    gg::derive_geometry(dimension_m, resolution, 0, k);
    float vx = point[0] - origin[0], vy = point[1] - origin[1], vz = point[2] - origin[2];
    const float sq = (vx * vx + vy * vy) + vz * vz;
    const float len = std::sqrt(sq);
    vx = vx / len;
    vy = vy / len;
    vz = vz / len;
    if (!(vz < -0.01f)) return -1;
    if (from < 0) return -1;
    const gg::OutlierRay ray{pos_xy[0], pos_xy[1], k.half, k.res, (double)len * (double)len, thr, tol, origin[0], origin[1], origin[2], vx, vy, vz, k.N};
    return gg::outlier_walk(ray, G, C, from > 2147483648LL ? 2147483648u : (unsigned)from) ? 1 : 0;
}

int gg_host_move_map(double res, double* pos_xy, double nx, double ny, int* shift_ij) {
    gg::move_map(res, pos_xy[0], pos_xy[1], nx, ny, shift_ij[0], shift_ij[1]);
    return (shift_ij[0] != 0 || shift_ij[1] != 0) ? 1 : 0;
}

// the resolve of k_pose_resolve (gg_internal.h:resolve_move) on the host: 1 moved, 0 not, -1 invalid (nothing written)
int gg_host_resolve_move(double res, double* pos_xy, double nx, double ny, int* shift_ij) {
    return gg::resolve_move(res, pos_xy[0], pos_xy[1], nx, ny, shift_ij[0], shift_ij[1]);
}

// out[9]: N, N2, full_layers, res_f, res, rres, len, half, res_sq
int gg_host_geometry_constants(double dimension_m, float resolution, unsigned flags, double* out) {
    gg::Const k;
    gg::derive_geometry(dimension_m, resolution, flags, k);
    const double v[9] = {(double)k.N, (double)k.N2, (double)k.full_layers, (double)k.res_f, k.res, k.rres, k.len, k.half, k.res_sq};
    std::memcpy(out, v, sizeof(v));
    return 0;
}

// out[16]: the fields of gg::CfgConst in declaration order (reserved left out)
int gg_host_config_constants(const gg_config* cfg, double* out) {
    gg::CfgConst k;
    gg::derive_config(*cfg, k);
    const double v[16] = {(double)k.max_ring, (double)k.pc_var_thresh_f, k.min_outlier_conf, k.outlier_tol, k.gp_thresh, k.df_sq, k.mdf_sq,
                          k.mdf10_sq, k.psc_sq, k.occ_factor, k.occ_factor2, k.dec_factor, k.lab_fac, k.lab_thres, k.lab_obs,
                          (double)k.decay_floor_ok};
    std::memcpy(out, v, sizeof(v));
    return 0;
}

// Replays configuration changes on a registry of n_slots slots that starts like a new handle (every slot on the
// default configuration).  Operation i sets op_cfg[i] on slot op_slot[i], or on the whole handle if op_slot[i] == -1;
// op_slot[i] = -2 - v marks variant v as holding unknown data (a failed build; op_cfg[i] is ignored).
// out: per operation (variant id of the slot or 0, 1 if the variant had to be built, live variants, variant ids),
// then the final variant of every slot.
int gg_host_config_registry(int n_slots, int n_ops, const int* op_slot, const gg_config* op_cfg, int* out) {
    if (n_slots <= 0 || n_ops < 0 || (n_ops && (!op_slot || !op_cfg)) || !out) return GG_E_ARG;
    gg::ConfigRegistry reg;
    gg_config c0;
    gg_default_config(&c0);
    gg::CfgConst k;
    gg::derive_config(c0, k);
    reg.reset(n_slots, k);
    for (int i = 0; i < n_ops; ++i) {
        if (op_slot[i] >= n_slots || (op_slot[i] <= -2 && -2 - op_slot[i] >= reg.ids())) return GG_E_ARG;
        gg::derive_config(op_cfg[i], k);
        int id = 0;
        bool build = true;
        if (op_slot[i] <= -2) {
            id = -2 - op_slot[i];
            build = false;
            reg.invalidate(id);
        } else if (op_slot[i] < 0)
            reg.reset(n_slots, k);
        else
            id = reg.assign(op_slot[i], k, &build);
        int* o = out + 4 * (size_t)i;
        o[0] = id;
        o[1] = build ? 1 : 0;
        o[2] = reg.live();
        o[3] = reg.ids();
    }
    for (int s = 0; s < n_slots; ++s) out[4 * (size_t)n_ops + s] = reg.variant_of(s);
    return 0;
}
}
