// C-ABI of groundgrid_b200 (include/groundgrid_b200.h): handle management, device arena,
// parameter staging, stream pipeline.  All compute happens in gg_kernels.cu; there is no CPU
// fallback -- without a usable sm_90 device every compute call returns GG_E_CUDA.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "gg_host.h"
#include "gg_internal.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define GG_CUDA(call)                                                                              \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess) return fail(GG_E_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

constexpr int kStreams = 8;   // upper bound; GG_STREAMS (default 8) picks how many are used
constexpr int kRing = 256;

// CUDA-event pairs around every kernel launch while profiling is enabled.
struct EventProfiler : gg::Profiler {
    struct Rec {
        int id;
        cudaEvent_t a, b;
    };
    std::vector<Rec> recs;
    std::vector<cudaEvent_t> pool;
    size_t dropped = 0;
    static constexpr size_t kMaxRecs = 16384;
    cudaEvent_t get() {
        if (!pool.empty()) {
            cudaEvent_t e = pool.back();
            pool.pop_back();
            return e;
        }
        cudaEvent_t e = nullptr;
        cudaEventCreate(&e);
        return e;
    }
    void begin(int id, cudaStream_t st) override {
        if (recs.size() >= kMaxRecs) {
            ++dropped;
            cur = nullptr;
            return;
        }
        recs.push_back({id, get(), get()});
        cur = &recs.back();
        cudaEventRecord(cur->a, st);
    }
    void end(int, cudaStream_t st) override {
        if (cur) cudaEventRecord(cur->b, st);
        cur = nullptr;
    }
    // after the streams were synchronised
    void collect(double* ms, uint32_t* count) {
        for (Rec& r : recs) {
            float t = 0.f;
            if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) {
                ms[r.id] += t;
                count[r.id] += 1;
            }
            pool.push_back(r.a);
            pool.push_back(r.b);
        }
        recs.clear();
    }
    ~EventProfiler() override {
        for (Rec& r : recs) {
            cudaEventDestroy(r.a);
            cudaEventDestroy(r.b);
        }
        for (cudaEvent_t e : pool) cudaEventDestroy(e);
    }
    Rec* cur = nullptr;
};

// Host-side packing of PointXYZIR clouds for the batched host-buffer path: the 32-byte records
// carry 14 useful bytes (x, y, z, ring); PCIe is the bottleneck of that path, so worker threads
// repack every cloud into pinned staging memory as x | y | z (float[n_pad]) | ring (u16[n_pad]), n_pad = n rounded up to 8,
// with streaming stores, and only 14 bytes per point cross the bus.
struct PackJob {
    const gg_point* src = nullptr;
    size_t n = 0;
    std::atomic<int> remaining{0};
};

class HostPacker {
  public:
    static constexpr size_t kChunk = 16384;  // points per work item (multiple of 8)
    explicit HostPacker(int threads) {
        for (int t = 0; t < threads; ++t) workers_.emplace_back([this] { loop(); });
    }
    ~HostPacker() {
        {
            std::lock_guard<std::mutex> g(mu_);
            stop_ = true;
            ++epoch_;
        }
        cv_.notify_all();
        for (auto& w : workers_) w.join();
    }
    int threads() const { return (int)workers_.size(); }

    // Staging ring: packed job number `seq` (counted over the lifetime of the handle) is written to slot
    // seq % slots.  The ring is small enough to stay in the last-level cache, so the packers' (plain) stores
    // and the DMA reads that follow mostly stay out of DRAM; a slot is reused once `copied` -- the number of
    // packed jobs whose H2D copy has completed, advanced by the feeding thread -- has passed its last user.
    void set_ring(unsigned char* base, size_t stride, int slots) {
        ring_ = base;
        stride_ = stride;
        slots_ = slots;
    }
    unsigned char* slot_of(uint64_t seq) const { return ring_ + (size_t)(seq % (uint64_t)slots_) * stride_; }
    std::atomic<uint64_t> copied{0};
    std::atomic<uint64_t> pack_ns{0}, slot_wait_ns{0};  // summed over the worker threads (diagnostics)

    // jobs must stay alive until every job is either packed or claimed raw (or cancel() has returned); chunks go
    // out in job order; job j is packed job number seq_base + j
    void start(std::vector<PackJob>* jobs, uint64_t seq_base) {
        while (busy_.load(std::memory_order_acquire) != 0) std::this_thread::yield();  // stragglers of the previous run
        std::vector<std::pair<int, int>> chunks;
        std::vector<size_t> first_chunk;
        for (size_t j = 0; j < jobs->size(); ++j) {
            PackJob& job = (*jobs)[j];
            const int nch = (int)std::max<size_t>(1, (job.n + kChunk - 1) / kChunk);
            job.remaining.store(nch, std::memory_order_relaxed);
            first_chunk.push_back(chunks.size());
            for (int c = 0; c < nch; ++c) chunks.push_back({(int)j, c});
        }
        {
            // everything a claim reads changes under the claim lock, so a worker that wakes up late sees either the
            // finished previous run (nothing to claim) or this one completely
            std::lock_guard<std::mutex> g(claim_mu_);
            chunks_.swap(chunks);
            first_chunk_.swap(first_chunk);
            jobs_ = jobs;
            seq_base_ = seq_base;
            next_ = 0;
            limit_ = chunks_.size();
            raw_from_ = (int)jobs->size();
            cancel_.store(false, std::memory_order_relaxed);
        }
        {
            std::lock_guard<std::mutex> g(mu_);
            ++epoch_;
        }
        cv_.notify_all();
    }
    // Error path of the caller: nothing more is claimed, chunks in flight are waited for; afterwards the job list
    // may be destroyed.
    void cancel() {
        {
            std::lock_guard<std::mutex> g(claim_mu_);
            limit_ = next_;
            cancel_.store(true, std::memory_order_release);
        }
        while (inflight_.load(std::memory_order_acquire) != 0) std::this_thread::yield();
    }
    // Take the last job nobody has started packing yet out of the packers' hands (it will be sent as
    // plain 32-byte records).  Returns its index or -1.
    int claim_raw_from_back() {
        std::lock_guard<std::mutex> g(claim_mu_);
        if (raw_from_ <= 0) return -1;
        const int j = raw_from_ - 1;
        if (first_chunk_[j] < next_) return -1;  // a packer is already on it
        raw_from_ = j;
        limit_ = first_chunk_[j];
        return j;
    }
    bool packed(const PackJob& job) const { return job.remaining.load(std::memory_order_acquire) <= 0; }
    bool help() { return work_one(false); }  // the calling thread packs one chunk if one can be started right away

    static void pack_range(const gg_point* src, size_t n, unsigned char* dst, size_t i0, size_t i1, bool cached = false) {
        gg::pack_cloud_range(src, n, dst, i0, i1, cached);
    }

  private:
    bool work_one(bool may_wait) {
        std::vector<PackJob>* jobs;
        size_t c;
        uint64_t seq;
        {
            std::lock_guard<std::mutex> g(claim_mu_);
            jobs = jobs_;
            if (!jobs || next_ >= limit_) return false;
            seq = seq_base_ + (uint64_t)chunks_[next_].first;
            if (!may_wait && seq >= copied.load(std::memory_order_acquire) + (uint64_t)slots_) return false;
            c = next_++;
            inflight_.fetch_add(1, std::memory_order_acq_rel);
        }
        const std::pair<int, int> chunk = chunks_[c];  // chunks_ only changes in start(), which waits for busy_ == 0
        const auto t0 = std::chrono::steady_clock::now();
        bool go = true;
        while (seq >= copied.load(std::memory_order_acquire) + (uint64_t)slots_) {  // the slot's previous cloud is still on its way
            if (stop_ || cancel_.load(std::memory_order_acquire)) {
                go = false;
                break;
            }
            std::this_thread::sleep_for(std::chrono::microseconds(20));
        }
        const auto t1 = std::chrono::steady_clock::now();
        if (go) {
            PackJob& job = (*jobs)[chunk.first];
            const size_t i0 = (size_t)chunk.second * kChunk;
            pack_range(job.src, job.n, slot_of(seq), i0, std::min(job.n, i0 + kChunk), true);
            job.remaining.fetch_sub(1, std::memory_order_release);
        }
        const auto t2 = std::chrono::steady_clock::now();
        slot_wait_ns.fetch_add((uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count(), std::memory_order_relaxed);
        pack_ns.fetch_add((uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t2 - t1).count(), std::memory_order_relaxed);
        inflight_.fetch_sub(1, std::memory_order_acq_rel);
        return go;
    }
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> g(mu_);
                cv_.wait(g, [&] { return epoch_ != seen; });
                seen = epoch_;
                if (stop_) return;
                busy_.fetch_add(1, std::memory_order_acq_rel);
            }
            while (work_one(true)) {
            }
            busy_.fetch_sub(1, std::memory_order_acq_rel);
        }
    }
    std::vector<std::thread> workers_;
    std::mutex mu_, claim_mu_;
    std::condition_variable cv_;
    std::vector<PackJob>* jobs_ = nullptr;
    std::vector<std::pair<int, int>> chunks_;
    std::vector<size_t> first_chunk_;
    unsigned char* ring_ = nullptr;
    size_t stride_ = 0;
    int slots_ = 1;
    uint64_t seq_base_ = 0;
    size_t next_ = 0, limit_ = 0;
    int raw_from_ = 0;
    std::atomic<int> busy_{0}, inflight_{0};
    std::atomic<bool> cancel_{false};
    uint64_t epoch_ = 0;
    std::atomic<bool> stop_{false};
};

struct SlotState {
    bool have_map = false;
    double px = 0.0, py = 0.0;
    size_t n_points = 0;       // points of the resident / last scan
    int last_stop = 0;         // stop_after of the last run (decides what "points" names)
    bool ran = false;
    bool output_valid = false;
    const gg_point* src = nullptr;  // caller-owned device cloud of the last scan (null: the slot's own buffer)
    const float* packed_input = nullptr;  // last scan came through the packed host path (no 32-byte records on the device)
    size_t scan_points = 0;    // points of the last scan (n_points may already count the next upload)
    bool moved_since_scan = false;  // a roll shifted the cells after the last scan: its cell indices are stale
    // gg_update_poses_from_device
    bool device_position = false;   // px / py are stale: the position lives in the device table (PoseTables::position)
    bool device_scan_pose = false;  // the device holds a scan pose of the slot (flagged scans may run)
    bool device_rolled = false;     // a device roll since the last scan (it may have moved the cells)
};

// A caller's device byte range [begin, end) of one query set: its positions (input) or one of its outputs.
struct ByteRange {
    uintptr_t begin, end;
    int set;
    bool output;
};

}  // namespace

struct gg_handle_s {
    int device = 0;
    int n_slots = 0;
    size_t pcap = 0;
    unsigned flags = 0;
    double dimension_m = 0.0;
    float resolution = 0.f;
    gg_config cfg{};                   // what gg_set_config last set (gg_get_config)
    std::vector<gg_config> slot_cfg;   // per slot: what gg_set_slot_config / gg_set_config last set
    gg::ConfigRegistry variants;       // slot -> configuration variant (shared by slots with identical constants)
    std::vector<float4*> variant_tab;  // per variant id: detect table of its constants (N2 entries)
    gg::View view{};
    std::vector<SlotState> slots;
    cudaStream_t streams[kStreams] = {};
    bool own_streams = true;
    int n_streams = kStreams;
    // parameter staging ring: pinned host copy + device copy per entry
    gg::SlotParams* h_ring = nullptr;
    gg::SlotParams* d_ring = nullptr;
    gg::OutDest* h_dest = nullptr;   // output destinations of the entry's scans, same shape as h_ring / d_ring
    gg::OutDest* d_dest = nullptr;
    gg::UnpackDesc* h_unpack = nullptr;  // PointCloud2 payloads of the entry's scans, same shape as h_ring / d_ring
    gg::UnpackDesc* d_unpack = nullptr;
    gg::QueryDesc* h_query = nullptr;    // terrain lookups: query sets of the entry's slots, same shape as h_ring / d_ring
    gg::QueryDesc* d_query = nullptr;
    gg::PointInfoDest* h_pinfo = nullptr;  // point classes and heights: destinations of the entry's slots, same shape
    gg::PointInfoDest* d_pinfo = nullptr;  // (both allocated on first use)
    int* h_pose_bits = nullptr;            // gg::PoseBits of the entry's records, same shape (allocated with `poses`)
    int* d_pose_bits = nullptr;
    gg::PoseTables poses{};                // per-slot device positions and scan poses (first gg_update_poses_from_device)
    cudaEvent_t ring_ev[kRing] = {};
    cudaEvent_t caller_in = nullptr;            // gg_run_scans_to_device: recorded on the caller's stream, awaited by the groups
    cudaEvent_t caller_out[kStreams] = {};      // ... recorded by each group after its outputs, awaited by the caller's stream
    bool ring_used[kRing] = {};
    int ring_pos = 0;
    uint64_t launches = 0;
    std::vector<void*> dev_allocs;
    std::vector<unsigned char> seen_scratch;  // duplicate-slot check of the batch calls (check_slots)
    std::vector<int> part_base;               // gg_run_merged_cloud_msgs_to_device: index in `parts` of each scan's first part
    std::vector<ByteRange> range_scratch;     // gg_sample_layers_to_device: the overlap check of the sets' ranges
    int sched_levels = 0, sched_visits = 0, sched_max = 0;
    bool out_cloud_ready = false;
    // f1: device copy of a PointCloud2 payload, one buffer per stream group (the copy and the unpack kernel of a slot
    // run on the slot's stream; stream order then keeps two slots of one group from overwriting each other's payload)
    unsigned char* d_raw[kStreams] = {};
    size_t d_raw_cap[kStreams] = {};
    float* d_image = nullptr;        // f3: terrain image staging (N * N * 3)
    unsigned char* d_image_u8 = nullptr;  // f3: 8-bit layer image staging (N * N)
    float* d_minmax = nullptr;       //     and its lower / upper
    int2* d_img_part = nullptr;      // f3: per-block ranges of the layer images, [n_slots][L_NUM][cdiv(N2, IMG_RANGE_CELLS)]
    unsigned long long* d_eval = nullptr;  // f4: [EVAL_LABELS][2] tallies
    HostPacker* packer = nullptr;    // created on the first packed batch call
    // gg_filter_cloud_batch[_begin] alternates between two sets of input / label buffers ("parity"), so the
    // clouds of batch t+1 can be packed and copied while the kernels of batch t still read theirs
    unsigned char* h_stage = nullptr;  // pinned staging ring of the packers, [pack_slots][14 * pcap] (HostPacker::set_ring)
    int pack_slots = 32;               // GG_PACK_RING
    std::vector<cudaEvent_t> slot_ev;  // [pack_slots] H2D of the slot's current cloud
    uint64_t pack_issued = 0;          // packed jobs whose copy has been enqueued (HostPacker::copied counts the completed ones)
    unsigned char* in_packed[2] = {};  // device, same shape
    gg_point* in_raw[2] = {};          // device 32-byte records; [0] is the slots' own buffer (view.points)
    uint8_t* labels_buf[2] = {};       // [0] is the buffer the handle was created with
    int batch_parity = 0;
    bool batch_outstanding[2] = {};
    cudaEvent_t batch_done[2] = {};    // on copy_out: kernels and label copies of the batch have finished
    int host_pack = 1;               // GG_HOST_PACK=0 sends the 32-byte records as they are
    int launch_unit = 32;            // GG_LAUNCH_UNIT: scans per kernel launch set in gg_filter_cloud_batch
    int host_pack_mix = 1;           // GG_HOST_PACK=1 pins "pack everything"; default: pack and send raw side by side
    cudaStream_t copy_in[10] = {}, copy_out = nullptr;  // [0, n_copy_in): packed clouds, then 2 for raw clouds;  // H2D / D2H of gg_filter_cloud_batch, never behind kernels
    int n_copy_in = 4;                                   // GG_COPY_STREAMS
    int main_help = 1;                                   // GG_MAIN_HELP
    CUtensorMap layer_map{};        // TMA descriptor of the layer arena (k_detect_tma); valid iff have_layer_map
    bool have_layer_map = false;
    bool inputs_busy = false;  // asynchronous work that reads or writes the slots' input buffers may be in flight
    std::vector<cudaEvent_t> batch_ev;                    // unit hand-over events of gg_filter_cloud_batch
    cudaEvent_t raw_ev[8] = {};      // throttle of the raw copies issued by the mixing loop
    int raw_gate = 2;                // GG_RAW_GATE (legacy, only with GG_BUS_TARGET_MB=0): no raw copies while this many packed clouds wait for the bus
    size_t bus_target = 8u << 20;    // GG_BUS_TARGET_MB: raw clouds are added while fewer bytes than this are in flight on the bus
    int raw_depth = 4;               // GG_RAW_DEPTH: raw copies in flight before the loop stops claiming more
    size_t last_raw = 0, last_packed = 0;  // scans sent raw / packed by the last batch call
    size_t last_raw_bytes = 0, last_packed_bytes = 0;
    size_t last_feed_us = 0, last_total_us = 0;
    size_t last_pack_us = 0, last_slot_wait_us = 0, last_idle_us = 0;  // worker-thread sums; feeder time with nothing to enqueue  // host time until the last cloud was enqueued / until everything was done
    EventProfiler* prof = nullptr;   // non-null while profiling is enabled
    double prof_ms[gg::K_NUM] = {};
    uint32_t prof_count[gg::K_NUM] = {};
};

namespace {

template <typename T>
int dev_alloc(gg_handle h, T** p, size_t count) {
    void* q = nullptr;
    GG_CUDA(cudaMalloc(&q, count * sizeof(T) + 256));
    h->dev_allocs.push_back(q);
    *p = static_cast<T*>(q);
    return GG_OK;
}

// a new device copy of src, with room for `pad` more elements (kernels that run ahead may read up to them)
template <typename T>
int dev_upload(gg_handle h, const T** p, const std::vector<T>& src, size_t pad = 0) {
    T* d = nullptr;
    int rc = dev_alloc(h, &d, src.size() + pad);
    if (rc) return rc;
    GG_CUDA(cudaMemcpy(d, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
    *p = d;
    return GG_OK;
}

int check_slot(gg_handle h, int slot) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (slot < 0 || slot >= h->n_slots) return fail(GG_E_ARG, "slot %d out of range [0, %d)", slot, h->n_slots);
    return GG_OK;
}

int layer_index(gg_handle h, int slot, const char* name, int* idx) {
    struct Entry {
        const char* name;
        int idx;
        bool full_only;
    };
    static const Entry table[] = {
        {"ground", gg::L_GROUND, false},        {"groundpatch", gg::L_GROUNDPATCH, false},
        {"variance", gg::L_VARIANCE, false},    {"minGroundHeight", gg::L_MINH, false},
        {"maxGroundHeight", gg::L_MAXH, true},  {"groundCandidates", gg::L_GCAND, true},
        {"planeDist", gg::L_PLANEDIST, true},   {"m2", gg::L_M2, true},
        {"meanVariance", gg::L_MEAN, true},     {"pointsRaw", gg::L_RAW, true},
        {"count", gg::L_COUNT, false},          {"obstacles", gg::L_OBSTACLES, false},
    };
    if (!name) return fail(GG_E_ARG, "null layer name");
    if (std::strcmp(name, "points") == 0) {
        // the reference reuses "points": kept-point count while rasterising (:309), non-ground
        // point count after the label loop (:147,176)
        const SlotState& s = h->slots[slot];
        *idx = (s.ran && s.last_stop != 0) ? gg::L_COUNT : gg::L_OBSTACLES;
        return GG_OK;
    }
    for (const Entry& e : table)
        if (std::strcmp(name, e.name) == 0) {
            if (e.full_only && !(h->flags & GG_FLAG_FULL_LAYERS)) return fail(GG_E_LAYER, "layer '%s' needs GG_FLAG_FULL_LAYERS", name);
            *idx = e.idx;
            return GG_OK;
        }
    return fail(GG_E_LAYER, "unknown layer '%s'", name);
}

// One entry of the parameter staging ring: the SlotParams of up to n_slots scans and, in arrays parallel to them, their
// output destinations (OutDest), PointCloud2 payloads (UnpackDesc), query sets (QueryDesc) and point-info destinations
// (PointInfoDest), each pinned on the host with a device copy.
struct Staging {
    int pos = 0;                 // position in the ring
    int m = 0;                   // records filled
    int max_points = 0;          // largest n_points of the records
    bool dests = false;          // commit also copies the OutDest records
    bool unpack = false;         // ... and the UnpackDesc records
    bool query = false;          // ... and the QueryDesc records
    bool pinfo = false;          // ... and the PointInfoDest records
    bool pose_bits = false;      // ... and the PoseBits of the records
    bool position = false;       // fill staged slot positions (run_groups then patches device-owned ones on the device)
    bool stage = false;          // some record takes its position or scan pose from the device tables (k_stage_poses)
    gg::SlotParams *hp = nullptr, *dp = nullptr;
    gg::OutDest *hdest = nullptr, *ddest = nullptr;
    gg::UnpackDesc *hunpack = nullptr, *dunpack = nullptr;
    gg::QueryDesc *hquery = nullptr, *dquery = nullptr;
    gg::PointInfoDest *hpinfo = nullptr, *dpinfo = nullptr;
    int *hbits = nullptr, *dbits = nullptr;

    // Reserve the next entry (waits only if the ring wrapped onto an in-flight entry).
    int acquire(gg_handle h) {
        pos = h->ring_pos;
        h->ring_pos = (pos + 1) % kRing;
        if (h->ring_used[pos]) GG_CUDA(cudaEventSynchronize(h->ring_ev[pos]));
        const size_t at = (size_t)pos * h->n_slots;
        hp = h->h_ring + at;
        dp = h->d_ring + at;
        hdest = h->h_dest + at;
        ddest = h->d_dest + at;
        hunpack = h->h_unpack + at;
        dunpack = h->d_unpack + at;
        hquery = h->h_query + at;
        dquery = h->d_query + at;
        hpinfo = h->h_pinfo ? h->h_pinfo + at : nullptr;   // allocated on the first gg_point_info_to_device
        dpinfo = h->d_pinfo ? h->d_pinfo + at : nullptr;
        hbits = h->h_pose_bits ? h->h_pose_bits + at : nullptr;   // allocated on the first gg_update_poses_from_device
        dbits = h->d_pose_bits ? h->d_pose_bits + at : nullptr;
        return GG_OK;
    }
    int commit(cudaStream_t st) const {
        GG_CUDA(cudaMemcpyAsync(dp, hp, (size_t)m * sizeof(gg::SlotParams), cudaMemcpyHostToDevice, st));
        if (dests) GG_CUDA(cudaMemcpyAsync(ddest, hdest, (size_t)m * sizeof(gg::OutDest), cudaMemcpyHostToDevice, st));
        if (unpack) GG_CUDA(cudaMemcpyAsync(dunpack, hunpack, (size_t)m * sizeof(gg::UnpackDesc), cudaMemcpyHostToDevice, st));
        if (query) GG_CUDA(cudaMemcpyAsync(dquery, hquery, (size_t)m * sizeof(gg::QueryDesc), cudaMemcpyHostToDevice, st));
        if (pinfo) GG_CUDA(cudaMemcpyAsync(dpinfo, hpinfo, (size_t)m * sizeof(gg::PointInfoDest), cudaMemcpyHostToDevice, st));
        if (pose_bits) GG_CUDA(cudaMemcpyAsync(dbits, hbits, (size_t)m * sizeof(int), cudaMemcpyHostToDevice, st));
        return GG_OK;
    }
    // The entry may be reused once the kernels that read it have finished (they may run on any of the handle's streams,
    // so the event is recorded AFTER the launches, not after the copy).
    int release(gg_handle h, cudaStream_t st) const {
        GG_CUDA(cudaEventRecord(h->ring_ev[pos], st));
        h->ring_used[pos] = true;
        return GG_OK;
    }
};

// Unpack descriptor of one payload whose layout has been validated (check_cloud_msg).
void fill_unpack(gg::UnpackDesc& d, const void* data, int point_step, const int field_offsets[5], const double* T_map_from_frame) {
    std::memset(&d, 0, sizeof(d));
    d.raw = static_cast<const unsigned char*>(data);
    d.point_step = point_step;
    for (int f = 0; f < 5; ++f) d.off[f] = field_offsets[f];
    d.transform = T_map_from_frame ? 1 : 0;
    if (T_map_from_frame) std::memcpy(d.T, T_map_from_frame, sizeof(d.T));
}

// The layout rules of a PointCloud2 payload: x, y, z present, every present field inside point_step.
int check_cloud_msg(const void* data, size_t n_points, int point_step, const int field_offsets[5]) {
    if ((n_points && !data) || !field_offsets || point_step < 12) return fail(GG_E_ARG, "bad PointCloud2 layout");
    for (int f = 0; f < 5; ++f) {
        const int width = f == 4 ? 2 : 4;
        if ((f < 3 && field_offsets[f] < 0) || field_offsets[f] + width > point_step) return fail(GG_E_ARG, "field %d does not fit point_step", f);
    }
    return GG_OK;
}

// Slots are bound to streams in contiguous groups; everything that touches a slot is enqueued
// on its stream, so scans of different groups overlap (the latency-bound spiral of one group
// runs under the bandwidth-bound kernels of another) without any cross-stream dependency.
int stream_index(gg_handle h, int slot) { return (int)((long long)slot * h->n_streams / h->n_slots); }
cudaStream_t stream_of(gg_handle h, int slot) { return h->streams[stream_index(h, slot)]; }

// The slots of a batched call: a list of slot ids, or the slots of a list of scans.
struct SlotList {
    const int* ids = nullptr;
    const gg_scan_desc* scans = nullptr;
    SlotList(const int* s) : ids(s) {}
    SlotList(const gg_scan_desc* s) : scans(s) {}
    int operator[](int i) const { return scans ? scans[i].slot : ids[i]; }
};

// The checks of every call on a list of slots, in this order: at most n_slots entries, then per entry a slot in range,
// no slot twice (the scans of a batch run concurrently), an initialised map and, for a list of scans, at most pcap points
// and (with `clouds`) a cloud for every non-empty scan.  h->seen_scratch is free again when it returns, so a checked call
// may run checked sub-batches.
int check_slots(gg_handle h, int count, SlotList slots, const gg_point* const* clouds = nullptr) {
    if (count > h->n_slots) return fail(GG_E_ARG, "count %d exceeds the number of slots %d", count, h->n_slots);
    std::vector<unsigned char>& seen = h->seen_scratch;
    seen.assign((size_t)h->n_slots, 0);
    int rc;
    for (int i = 0; i < count; ++i) {
        const int slot = slots[i];
        if ((rc = check_slot(h, slot))) return rc;
        if (seen[slot]++) return fail(GG_E_ARG, "slot %d appears twice in one batch (scans of a batch run concurrently)", slot);
        if (!h->slots[slot].have_map) return fail(GG_E_STATE, "slot %d: map not initialised", slot);
        if (!slots.scans) continue;
        if ((slots.scans[i].flags & GG_SCAN_DEVICE_POSE) && !h->slots[slot].device_scan_pose)
            return fail(GG_E_STATE, "slot %d: GG_SCAN_DEVICE_POSE without a device scan pose since gg_init_map", slot);
        const size_t n = slots.scans[i].n_points;
        if (n > h->pcap) return fail(GG_E_ARG, "slot %d: %zu points exceed capacity %zu", slot, n, h->pcap);
        if (clouds && n && !clouds[i]) return fail(GG_E_ARG, "scan %d: null cloud", i);
    }
    return GG_OK;
}

// Every launch of a batch goes through here.  Per stream group with scans in the batch, on the group's stream: one
// staging entry, fill(i, entry) for each of the group's scans i (it fills record entry.m and returns whether the record
// needs the device), the copy of the entry, launch(entry, stream) (returns the number of kernels it launched, or a
// negative error code), and the
// release of the entry.  A group whose records need nothing (a roll that moves no slot) only takes and releases its
// entry.  With `fenced`, the groups start after everything enqueued on `caller` so far, and `caller` waits for them: no
// host wait but the flow control of the staging ring.
// Poses: when fill staged slot positions (e.position), a record of a slot whose position is device-owned, or of a scan
// flagged GG_SCAN_DEVICE_POSE, is patched from the device tables by k_stage_poses right after the copy.  Without such
// records (every all-host flow) nothing more is copied or launched.
template <typename Fill, typename Launch>
int run_groups(gg_handle h, int count, SlotList slots, bool fenced, cudaStream_t caller, Fill&& fill, Launch&& launch) {
    int rc;
    if (fenced) GG_CUDA(cudaEventRecord(h->caller_in, caller));
    for (int g = 0; g < h->n_streams; ++g) {
        Staging e;
        bool work = false;
        for (int i = 0; i < count; ++i) {
            if (stream_index(h, slots[i]) != g) continue;
            if (e.m == 0 && (rc = e.acquire(h))) return rc;
            work |= fill(i, e);
            if (e.position && e.hbits) {
                int bits = h->slots[slots[i]].device_position ? gg::POSE_POSITION : 0;
                if (slots.scans && (slots.scans[i].flags & GG_SCAN_DEVICE_POSE)) bits |= gg::POSE_ORIGIN;
                e.hbits[e.m] = bits;
                if (bits) e.stage = e.pose_bits = true;
            }
            e.max_points = std::max(e.max_points, e.hp[e.m].n_points);
            ++e.m;
        }
        if (e.m == 0) continue;
        cudaStream_t st = h->streams[g];
        if (work) {
            if ((rc = e.commit(st))) return rc;
            if (e.stage) h->launches += gg::launch_stage_poses(h->poses, e.dp, e.dbits, e.m, st, h->prof);
            if (fenced) GG_CUDA(cudaStreamWaitEvent(st, h->caller_in, 0));
            const int n = launch(e, st);
            if (n < 0) return n;
            h->launches += n;
            GG_CUDA(cudaGetLastError());
        }
        if ((rc = e.release(h, st))) return rc;
        if (fenced) {
            GG_CUDA(cudaEventRecord(h->caller_out[g], st));
            GG_CUDA(cudaStreamWaitEvent(caller, h->caller_out[g], 0));
        }
    }
    return GG_OK;
}

// Device buffer of variant id `id` (allocated once, kept for reuse by later variants).
int ensure_variant_buffer(gg_handle h, int id) {
    int rc;
    while ((int)h->variant_tab.size() <= id) {
        float4* p = nullptr;
        if ((rc = dev_alloc(h, &p, (size_t)h->view.k.N2))) return rc;
        h->variant_tab.push_back(p);
    }
    return GG_OK;
}

// Device data of variant `id` (its detect table) from its constants on `st`, then a wait on `st`, so that every stream
// may use the variant afterwards.  Only called for a variant no enqueued work reads.
int build_variant(gg_handle h, int id, cudaStream_t st) {
    int rc;
    if ((rc = ensure_variant_buffer(h, id))) return rc;
    h->launches += gg::launch_build_detect_table(h->view, h->variants.constants(id), h->variant_tab[id], st);
    GG_CUDA(cudaGetLastError());
    GG_CUDA(cudaStreamSynchronize(st));
    return GG_OK;
}

void fill_params(gg_handle h, const gg_scan_desc& d, gg::SlotParams& p, const gg_point* src, const float* packed = nullptr) {
    const SlotState& s = h->slots[d.slot];
    std::memset(&p, 0, sizeof(p));
    const int var = h->variants.variant_of(d.slot);
    p.cfg = h->variants.constants(var);
    p.detect_tab = h->variant_tab[var];
    p.px = s.px;
    p.py = s.py;
    p.ox = d.origin[0];
    p.oy = d.origin[1];
    p.oz = d.origin[2];
    p.base_z_f = (float)d.base_z;  // ggl(c, c) = ps.point.z (double -> float), GroundSegmentation.cpp:411
    p.n_points = (int)d.n_points;
    p.slot = d.slot;
    p.src = src ? src : h->view.points + (size_t)d.slot * h->pcap;
    p.packed = packed;
}

// Caller-owned destinations of gg_run_scans_to_device / gg_run_cloud_msgs_to_device (validated by them) and the
// caller's stream.
struct CallerOutputs {
    const gg_scan_outputs* outs;  // [count] or null
    unsigned select;
    int32_t* counts;              // [count] or null
    cudaStream_t stream;
    const gg_cloud_msg* msgs;     // [count] or null: payloads unpacked into the slots' own buffers before the scans
    // or, for merged scans (validated by gg_run_merged_cloud_msgs_to_device), the n_parts[k] payloads of scan k at
    // parts + part_base[k]
    const int* n_parts = nullptr;
    const gg_cloud_part* parts = nullptr;
    const int* part_base = nullptr;
};

// A staging entry per part round is taken while the group's scan entry is held, so the rounds of one group never
// wrap the ring onto it.
static_assert(GG_MAX_CLOUD_PARTS < kRing, "the part rounds of a group must fit in the staging ring");

// The part rounds of the merged scans in the scan entry `e` (e.hp[j].pos = the scan's position in the call), on the
// group's stream `st`: round p is one launch of the unpack kernel over part p of every scan of the group that has a
// non-empty one, each landing in its slot's buffer after the scan's parts before p.  Each round takes its own staging
// entry.  Returns the number of launches, or a negative error code.
int launch_part_rounds(gg_handle h, const Staging& e, const CallerOutputs& c, cudaStream_t st) {
    int rounds = 0, n = 0, rc;
    for (int j = 0; j < e.m; ++j) rounds = std::max(rounds, c.n_parts[e.hp[j].pos]);
    for (int p = 0; p < rounds; ++p) {
        Staging r;
        for (int j = 0; j < e.m; ++j) {
            const int k = e.hp[j].pos;
            if (p >= c.n_parts[k]) continue;
            const gg_cloud_part* part = c.parts + c.part_base[k];
            if (part[p].n_points == 0) continue;
            if (r.m == 0 && (rc = r.acquire(h))) return rc;
            gg::SlotParams& sp = r.hp[r.m];
            std::memset(&sp, 0, sizeof(sp));
            sp.slot = e.hp[j].slot;
            sp.n_points = (int)part[p].n_points;
            const gg_cloud_msg& msg = part[p].msg;
            fill_unpack(r.hunpack[r.m], msg.data, msg.point_step, msg.field_offsets, msg.T_map_from_frame);
            size_t first = 0;
            for (int q = 0; q < p; ++q) first += part[q].n_points;
            r.hunpack[r.m].first = (int)first;
            r.max_points = std::max(r.max_points, sp.n_points);
            ++r.m;
        }
        if (r.m == 0) continue;
        r.unpack = true;
        if ((rc = r.commit(st))) return rc;
        n += gg::launch_unpack(h->view, r.dp, r.dunpack, r.m, r.max_points, st, h->prof);
        GG_CUDA(cudaGetLastError());
        if ((rc = r.release(h, st))) return rc;
    }
    return n;
}

// enqueue the kernels of `count` scans, each group of slots on its own stream; with `caller`, each group also writes
// its scans' outputs and is ordered after / before the caller's stream (and, with caller->msgs or caller->parts, first
// unpacks its scans' payloads)
int run_scans_grouped(gg_handle h, int count, const gg_scan_desc* scans, int stop_after, const gg_point* const* dev_points = nullptr,
                      const float* const* packed_ptrs = nullptr, uint8_t* labels_base = nullptr, const CallerOutputs* caller = nullptr) {
    if (count <= 0) return GG_OK;
    int rc;
    if ((rc = check_slots(h, count, scans))) return rc;
    gg::View view = h->view;
    if (labels_base) view.labels = labels_base;
    // count + scan passes when counts are wanted; the write pass when any scan of the group wants labels, index or cloud
    const bool compact = caller && caller->counts && caller->select;
    bool write = false;
    auto fill = [&](int i, Staging& e) {
        const gg_scan_desc& d = scans[i];
        const float* packed = packed_ptrs ? packed_ptrs[i] : nullptr;
        fill_params(h, d, e.hp[e.m], dev_points ? dev_points[i] : nullptr, packed);
        e.position = true;
        if (caller) {
            if (e.m == 0) write = false;
            gg::OutDest& od = e.hdest[e.m];
            std::memset(&od, 0, sizeof(od));
            if (caller->outs) {
                od.labels = caller->outs[i].labels;
                od.index = caller->outs[i].index;
                od.cloud = caller->outs[i].cloud;
            }
            od.count = compact ? caller->counts + i : nullptr;
            od.select = caller->select;
            write = write || od.labels || od.index || od.cloud;
            e.dests = compact || write;
            if (caller->msgs) {
                const gg_cloud_msg& msg = caller->msgs[i];
                fill_unpack(e.hunpack[e.m], msg.data, msg.point_step, msg.field_offsets, msg.T_map_from_frame);
                e.unpack = true;
            }
            if (caller->parts) e.hp[e.m].pos = i;
        }
        SlotState& s = h->slots[d.slot];
        s.n_points = d.n_points;
        s.last_stop = stop_after;
        s.ran = true;
        s.output_valid = false;
        s.src = dev_points ? dev_points[i] : nullptr;
        s.packed_input = packed;
        s.scan_points = d.n_points;
        s.moved_since_scan = false;
        s.device_rolled = false;
        return true;
    };
    auto launch = [&](const Staging& e, cudaStream_t st) {
        int n = 0;
        // after the wait on the caller's stream: the payloads may be produced there
        if (e.unpack) n += gg::launch_unpack(view, e.dp, e.dunpack, e.m, e.max_points, st, h->prof);
        if (caller && caller->parts) {
            const int r = launch_part_rounds(h, e, *caller, st);
            if (r < 0) return r;
            n += r;
        }
        n += gg::launch_scan_pipeline(view, e.dp, e.m, e.max_points, stop_after, st, h->prof, h->have_layer_map ? &h->layer_map : nullptr);
        if (e.dests) n += gg::launch_output(view, e.dp, e.ddest, e.m, e.max_points, compact, write, st, h->prof);
        return n;
    };
    return run_groups(h, count, scans, caller != nullptr, caller ? caller->stream : nullptr, fill, launch);
}

// TMA descriptor of the layer arena seen as a 3-D fp32 tensor (i fastest, j, plane = slot * n_layers + layer), box
// 40 x 12 x 1 = the halo tile of k_detect_tma (the box starts at i0 - 4: TMA wants a 16-byte aligned innermost start).  cuTensorMapEncodeTiled is a driver-API call; it is resolved through the
// runtime (cudaGetDriverEntryPoint) so that the library needs no link-time libcuda.  Row pitch must be a multiple of
// 16 bytes: maps with N % 4 != 0 keep the plain-load kernel.
bool encode_layer_map(gg_handle h) {
    const gg::View& v = h->view;
    if (v.k.N % 4 != 0) return false;
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
        cudaGetLastError();
        return false;
    }
    const cuuint64_t dims[3] = {(cuuint64_t)v.k.N, (cuuint64_t)v.k.N, (cuuint64_t)h->n_slots * (cuuint64_t)v.n_layers};
    const cuuint64_t strides[2] = {(cuuint64_t)v.k.N * sizeof(float), (cuuint64_t)v.k.N2 * sizeof(float)};
    const cuuint32_t box[3] = {40u, 12u, 1u};   // DT_WT x DT_R of k_detect_tma
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    const CUresult r = reinterpret_cast<EncodeFn>(fn)(&h->layer_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, v.layers, dims, strides, box, estr,
                                                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

int ensure_out_cloud(gg_handle h) {
    if (h->out_cloud_ready) return GG_OK;
    int rc = dev_alloc(h, &h->view.out_cloud, (size_t)h->n_slots * h->pcap);
    if (rc) return rc;
    h->out_cloud_ready = true;
    return GG_OK;
}

int run_output_on(gg_handle h, int slot, bool want_cloud) {
    SlotState& s = h->slots[slot];
    if (!s.ran || s.last_stop != 0) return fail(GG_E_STATE, "slot %d: no completed scan", slot);
    if (want_cloud && s.packed_input)
        return fail(GG_E_STATE, "slot %d: the output cloud needs the 32-byte records on the device (use gg_filter_cloud or GG_HOST_PACK=0)", slot);
    int rc;
    if (want_cloud && (rc = ensure_out_cloud(h))) return rc;
    auto fill = [&](int, Staging& e) {
        gg::SlotParams& p = e.hp[0];
        std::memset(&p, 0, sizeof(p));
        p.slot = slot;
        p.n_points = (int)s.n_points;
        p.src = s.src ? s.src : h->view.points + (size_t)slot * h->pcap;
        gg::OutDest& od = e.hdest[0];
        std::memset(&od, 0, sizeof(od));
        od.index = h->view.out_index + (size_t)slot * h->pcap;
        od.cloud = want_cloud ? h->view.out_cloud + (size_t)slot * h->pcap : nullptr;
        od.select = GG_SELECT_GROUND | GG_SELECT_NONGROUND;
        e.dests = true;
        return true;
    };
    auto launch = [&](const Staging& e, cudaStream_t st) { return gg::launch_output(h->view, e.dp, e.ddest, 1, e.max_points, true, true, st, h->prof); };
    if ((rc = run_groups(h, 1, &slot, false, nullptr, fill, launch))) return rc;
    s.output_valid = true;
    return GG_OK;
}

// The layer "points" names for `slot` (layer_index without the name lookup).
int points_layer(gg_handle h, int slot) {
    int idx = 0;
    layer_index(h, slot, "points", &idx);
    return idx;
}

// The batched calls on a list of slots and layer names: one staging record per slot (p.slot, p.pos = its position in the
// call, p.points_layer), each stream group ordered after / before `stream`.
template <typename Launch>
int enqueue_slot_batch(gg_handle h, int count, const int* slots, void* stream, Launch&& launch) {
    GG_CUDA(cudaSetDevice(h->device));
    auto fill = [&](int i, Staging& e) {
        gg::SlotParams& p = e.hp[e.m];
        std::memset(&p, 0, sizeof(p));
        p.slot = slots[i];
        p.pos = i;
        p.points_layer = points_layer(h, slots[i]);
        return true;
    };
    return run_groups(h, count, slots, true, static_cast<cudaStream_t>(stream), fill, launch);
}

// One phase of the slot's pipeline: a one-scan batch of its last scan on the slot's stream
template <typename Launch>
int run_phase(gg_handle h, int slot, double base_z, Launch&& launch) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!h->slots[slot].have_map) return fail(GG_E_STATE, "slot %d: map not initialised", slot);
    GG_CUDA(cudaSetDevice(h->device));
    auto fill = [&](int, Staging& e) {
        gg_scan_desc d;
        std::memset(&d, 0, sizeof(d));
        d.slot = slot;
        d.n_points = h->slots[slot].n_points;
        d.base_z = base_z;
        fill_params(h, d, e.hp[0], h->slots[slot].src);
        e.position = true;
        return true;
    };
    return run_groups(h, 1, &slot, false, nullptr, fill, launch);
}

// A call that needs the map position on the host: a device-owned position is read back once the slot's stream group
// has finished what is enqueued (a host wait), and the slot is host-owned again.
int take_position_back(gg_handle h, int slot) {
    SlotState& s = h->slots[slot];
    if (!s.device_position) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream_of(h, slot);
    double2 p;
    GG_CUDA(cudaMemcpyAsync(&p, h->poses.position + slot, sizeof(p), cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaStreamSynchronize(st));
    s.px = p.x;
    s.py = p.y;
    s.device_position = false;
    return GG_OK;
}

}  // namespace

extern "C" {

void gg_default_config(gg_config* c) {
    if (!c) return;
    c->point_count_cell_variance_threshold = 10;
    c->max_ring = 1024;
    c->groundpatch_detection_minimum_threshold = 0.01;
    c->distance_factor = 0.0001;
    c->minimum_distance_factor = 0.0005;
    c->miminum_point_height_threshold = 0.3;
    c->minimum_point_height_obstacle_threshold = 0.1;
    c->outlier_tolerance = 0.1;
    c->ground_patch_detection_minimum_point_count_threshold = 0.25;
    c->patch_size_change_distance = 20.0;
    c->occupied_cells_decrease_factor = 5.0;
    c->occupied_cells_point_count_factor = 20.0;
    c->min_outlier_detection_ground_confidence = 1.25;
    c->thread_count = 8;
}

const char* gg_last_error(void) { return g_last_error.c_str(); }

int gg_create(double dimension_m, float resolution, int device, int n_slots, size_t max_points, unsigned flags, void* stream,
              gg_handle* out) {
    if (!out) return fail(GG_E_ARG, "null out pointer");
    *out = nullptr;
    if (n_slots <= 0 || max_points == 0 || !(resolution > 0.f) || !(dimension_m > 0.0)) return fail(GG_E_ARG, "bad geometry / sizes");
    if (max_points > (1u << 26) - 256) return fail(GG_E_ARG, "max_points above 2^26 per cloud is not supported");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
        return fail(GG_E_CUDA, "no CUDA device available (groundgrid_b200 has no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(GG_E_ARG, "device %d out of range", device);
    cudaDeviceProp prop;
    GG_CUDA(cudaGetDeviceProperties(&prop, device));
    // sm_90a code runs on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0)
        return fail(GG_E_CUDA, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    GG_CUDA(cudaSetDevice(device));

    const int n = gg::cells_per_side(dimension_m, resolution);
    if (n < 8 || n > 4096) return fail(GG_E_ARG, "unsupported map size %d cells", n);

    gg_handle h = new gg_handle_s();
    h->device = device;
    h->n_slots = n_slots;
    h->pcap = (max_points + 255) / 256 * 256;
    h->flags = flags;
    h->dimension_m = dimension_m;
    h->resolution = resolution;
    gg_default_config(&h->cfg);
    h->slots.resize(n_slots);
    h->slot_cfg.assign((size_t)n_slots, h->cfg);
    {
        gg::CfgConst kc;
        gg::derive_config(h->cfg, kc);
        h->variants.reset(n_slots, kc);
    }
    gg::View& v = h->view;
    gg::derive_geometry(dimension_m, resolution, flags, v.k);
    if (v.k.N != n) {
        const int n_geo = v.k.N;
        delete h;
        return fail(GG_E_ARG, "cell count mismatch between init (%d) and setGeometry (%d)", n, n_geo);
    }
    const size_t N2 = (size_t)v.k.N2;
    v.n_layers = (flags & GG_FLAG_FULL_LAYERS) ? gg::L_NUM : gg::L_NUM_LIVE;
    v.pcap = h->pcap;
    v.out_blocks = (int)((h->pcap + gg::OUT_TILE - 1) / gg::OUT_TILE);

#define GG_TRY(expr)            \
    do {                        \
        int rc__ = (expr);      \
        if (rc__) {             \
            gg_destroy(h);      \
            return rc__;        \
        }                       \
    } while (0)
#define GG_CUDA_TRY(call)                                                                             \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess) {                                                                     \
            gg_destroy(h);                                                                            \
            return fail(GG_E_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
        }                                                                                             \
    } while (0)

    const size_t S = (size_t)n_slots, P = h->pcap;
    GG_TRY(dev_alloc(h, &v.layers, S * v.n_layers * N2));
    h->have_layer_map = encode_layer_map(h);
    float* expected = nullptr;
    GG_TRY(dev_alloc(h, &expected, N2));
    v.expected = expected;
    GG_TRY(dev_alloc(h, &v.points, S * P));
    GG_TRY(dev_alloc(h, &v.zw, S * P));
    GG_TRY(dev_alloc(h, &v.zsorted, S * P));
    GG_TRY(dev_alloc(h, &v.runj, S * P));
    GG_TRY(dev_alloc(h, &v.rundir, S * P));
    GG_TRY(dev_alloc(h, &v.dist, S * P));
    GG_TRY(dev_alloc(h, &v.code, S * P));
    GG_TRY(dev_alloc(h, &v.labels, S * P));
    GG_TRY(dev_alloc(h, &v.cnt64, S * N2));
    GG_TRY(dev_alloc(h, &v.raw_i, (flags & GG_FLAG_FULL_LAYERS) ? S * N2 : 1));
    GG_TRY(dev_alloc(h, &v.cellstart, S * N2));
    GG_TRY(dev_alloc(h, &v.worklist, S * N2));
    GG_TRY(dev_alloc(h, &v.wl_count, 2 * S));
    v.cell_tiles = (int)((N2 + 4095) / 4096);
    GG_TRY(dev_alloc(h, &v.cell_agg, S * v.cell_tiles * 65));
    GG_TRY(dev_alloc(h, &v.out_index, S * P));
    GG_TRY(dev_alloc(h, &v.out_counts, S * (3 * (size_t)v.out_blocks + 1)));
    GG_TRY(dev_alloc(h, &v.roll_scratch, S * 2 * N2));
    v.out_cloud = nullptr;
    GG_CUDA_TRY(cudaMemset(v.layers, 0, S * v.n_layers * N2 * sizeof(float)));
    // per-cell counters are zero between scans (k_cell_stats resets what it consumed)
    GG_CUDA_TRY(cudaMemset(v.cnt64, 0, S * N2 * sizeof(unsigned long long)));
    if (flags & GG_FLAG_FULL_LAYERS) GG_CUDA_TRY(cudaMemset(v.raw_i, 0, S * N2 * sizeof(int)));

    // expectedPoints table (host libm, like the reference) and the tables of the spiral path (gg_host.cpp:plan_spiral)
    {
        std::vector<float> table;
        gg::build_expected_points(n, table);
        GG_CUDA_TRY(cudaMemcpy(expected, table.data(), N2 * sizeof(float), cudaMemcpyHostToDevice));
        gg::SpiralPlan plan;
        gg::plan_spiral(n, v.k.res_sq, plan);
        GG_TRY(dev_upload(h, &v.level_start, plan.level_start));
        GG_TRY(dev_upload(h, &v.visits, plan.visits, 1));
        v.levels = (int)plan.level_start.size() - 1;
        h->sched_levels = v.levels;
        h->sched_visits = (int)plan.visits.size();
        h->sched_max = plan.max_per_level;
        v.spiral_threads = plan.threads;
        v.spiral_recs = nullptr;
        std::memset(&v.skew, 0, sizeof(v.skew));
        if (plan.kind == gg::SPIRAL_PIPE) {
            const uint32_t* d_rc = nullptr;
            GG_TRY(dev_upload(h, &d_rc, plan.recs, 4));
            v.spiral_recs = reinterpret_cast<const uint4*>(d_rc);
        } else if (plan.kind == gg::SPIRAL_SKEW) {
            const gg::SkewTables& sk = plan.skew;
            gg::SkewView& w = v.skew;
            GG_TRY(dev_upload(h, &w.ph_begin, plan.ph_begin));
            GG_TRY(dev_upload(h, &w.ph_end, plan.ph_end));
            GG_TRY(dev_upload(h, &w.ph_cell0, plan.ph_cell0));
            GG_TRY(dev_upload(h, &w.cell_home, sk.cell_home));
            const uint32_t* d_irr = nullptr;
            GG_TRY(dev_upload(h, &d_irr, plan.irr_blocks, 16));
            float2* d_sk = nullptr;
            float* d_sd = nullptr;
            GG_TRY(dev_alloc(h, &d_sk, S * sk.slots));
            GG_TRY(dev_alloc(h, &d_sd, S * sk.slots));
            GG_CUDA_TRY(cudaMemset(d_sk, 0, S * sk.slots * sizeof(float2)));
            GG_CUDA_TRY(cudaMemset(d_sd, 0, S * sk.slots * sizeof(float)));
            w.sk = d_sk;
            w.sd = d_sd;
            w.slots = sk.slots;
            w.M = plan.M;
            w.phases = plan.phases;
            w.irr_blocks = reinterpret_cast<const uint4*>(d_irr);
            w.irr_max = plan.irr_max;
            w.irr_chunks = plan.irr_chunks;
            w.KP = sk.KP;
            w.rows = sk.rows;
            w.row0 = sk.row0;
            w.lanes = sk.lanes;
            w.levels = sk.levels;
            std::memcpy(w.pattern, sk.pattern, sizeof(sk.pattern));
        }
    }

    if (const char* e = getenv("GG_LAUNCH_UNIT")) h->launch_unit = std::max(1, atoi(e));
    if (const char* e = getenv("GG_COPY_STREAMS")) h->n_copy_in = std::min(8, std::max(1, atoi(e)));
    if (const char* e = getenv("GG_MAIN_HELP")) h->main_help = atoi(e);
    if (const char* e = getenv("GG_RAW_GATE")) h->raw_gate = std::max(1, atoi(e));
    if (const char* e = getenv("GG_BUS_TARGET_MB")) h->bus_target = (size_t)std::max(0, atoi(e)) << 20;
    if (const char* e = getenv("GG_RAW_DEPTH")) h->raw_depth = std::min(8, std::max(1, atoi(e)));
    if (const char* e = getenv("GG_HOST_PACK")) {
        h->host_pack = atoi(e) ? 1 : 0;
        h->host_pack_mix = 0;
    }
    v.packed = nullptr;
    if (stream) {
        h->own_streams = false;
        h->n_streams = 1;
        h->streams[0] = static_cast<cudaStream_t>(stream);
    } else {
        int want = 8;
        if (const char* e = getenv("GG_STREAMS")) want = atoi(e);
        h->n_streams = std::max(1, std::min(std::min(want, kStreams), n_slots));
        for (int i = 0; i < h->n_streams; ++i) GG_CUDA_TRY(cudaStreamCreateWithFlags(&h->streams[i], cudaStreamNonBlocking));
    }
    GG_CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&h->h_ring), sizeof(gg::SlotParams) * kRing * S, cudaHostAllocDefault));
    GG_TRY(dev_alloc(h, &h->d_ring, (size_t)kRing * S));
    GG_CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&h->h_dest), sizeof(gg::OutDest) * kRing * S, cudaHostAllocDefault));
    GG_TRY(dev_alloc(h, &h->d_dest, (size_t)kRing * S));
    GG_CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&h->h_unpack), sizeof(gg::UnpackDesc) * kRing * S, cudaHostAllocDefault));
    GG_TRY(dev_alloc(h, &h->d_unpack, (size_t)kRing * S));
    GG_CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(&h->h_query), sizeof(gg::QueryDesc) * kRing * S, cudaHostAllocDefault));
    GG_TRY(dev_alloc(h, &h->d_query, (size_t)kRing * S));
    for (int i = 0; i < kRing; ++i) GG_CUDA_TRY(cudaEventCreateWithFlags(&h->ring_ev[i], cudaEventDisableTiming));
    GG_CUDA_TRY(cudaEventCreateWithFlags(&h->caller_in, cudaEventDisableTiming));
    for (int i = 0; i < kStreams; ++i) GG_CUDA_TRY(cudaEventCreateWithFlags(&h->caller_out[i], cudaEventDisableTiming));
    GG_TRY(build_variant(h, 0, h->streams[0]));
#undef GG_TRY
#undef GG_CUDA_TRY
    *out = h;
    return GG_OK;
}

int gg_destroy(gg_handle h) {
    if (!h) return GG_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    delete h->prof;
    delete h->packer;
    for (int g = 0; g < kStreams; ++g)
        if (h->d_raw[g]) cudaFree(h->d_raw[g]);
    if (h->h_stage) cudaFreeHost(h->h_stage);
    for (cudaEvent_t e : h->slot_ev) cudaEventDestroy(e);
    for (int i = 0; i < kStreams; ++i)
        if (h->caller_out[i]) cudaEventDestroy(h->caller_out[i]);
    if (h->caller_in) cudaEventDestroy(h->caller_in);
    for (int e = 0; e < 2; ++e)
        if (h->batch_done[e]) cudaEventDestroy(h->batch_done[e]);
    for (int e = 0; e < 8; ++e)
        if (h->raw_ev[e]) cudaEventDestroy(h->raw_ev[e]);
    for (cudaEvent_t e : h->batch_ev) cudaEventDestroy(e);
    for (int e = 0; e < 10; ++e)
        if (h->copy_in[e]) cudaStreamDestroy(h->copy_in[e]);
    if (h->copy_out) cudaStreamDestroy(h->copy_out);
    for (void* p : h->dev_allocs) cudaFree(p);
    if (h->h_ring) cudaFreeHost(h->h_ring);
    if (h->h_dest) cudaFreeHost(h->h_dest);
    if (h->h_unpack) cudaFreeHost(h->h_unpack);
    if (h->h_query) cudaFreeHost(h->h_query);
    if (h->h_pinfo) cudaFreeHost(h->h_pinfo);
    if (h->h_pose_bits) cudaFreeHost(h->h_pose_bits);
    for (int i = 0; i < kRing; ++i)
        if (h->ring_ev[i]) cudaEventDestroy(h->ring_ev[i]);
    if (h->own_streams)
        for (int i = 0; i < h->n_streams; ++i)
            if (h->streams[i]) cudaStreamDestroy(h->streams[i]);
    delete h;
    return GG_OK;
}

int gg_cells_per_side(gg_handle h) { return h ? h->view.k.N : GG_E_ARG; }
int gg_num_slots(gg_handle h) { return h ? h->n_slots : GG_E_ARG; }
void* gg_stream(gg_handle h) { return h ? h->streams[0] : nullptr; }
uint64_t gg_kernel_launches(gg_handle h) { return h ? h->launches : 0; }

int gg_spiral_schedule_info(gg_handle h, int* levels, int* visits, int* max_per_level) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (levels) *levels = h->sched_levels;
    if (visits) *visits = h->sched_visits;
    if (max_per_level) *max_per_level = h->sched_max;
    return GG_OK;
}

int gg_set_config(gg_handle h, const gg_config* cfg) {
    if (!h || !cfg) return fail(GG_E_ARG, "null argument");
    GG_CUDA(cudaSetDevice(h->device));
    int rc = gg_synchronize(h);  // kernels in flight keep the tables of the old configuration
    if (rc) return rc;
    h->cfg = *cfg;
    h->slot_cfg.assign((size_t)h->n_slots, *cfg);
    gg::CfgConst kc;
    gg::derive_config(*cfg, kc);
    h->variants.reset(h->n_slots, kc);   // every slot on variant 0; nothing reads the others any more
    return build_variant(h, 0, h->streams[0]);
}

int gg_get_config(gg_handle h, gg_config* cfg) {
    if (!h || !cfg) return fail(GG_E_ARG, "null argument");
    *cfg = h->cfg;
    return GG_OK;
}

int gg_set_slot_config(gg_handle h, int slot, const gg_config* cfg) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!cfg) return fail(GG_E_ARG, "null argument");
    GG_CUDA(cudaSetDevice(h->device));
    // Every kernel that reads the slot's variant runs on the slot's stream: once that stream is idle, the old variant
    // is read by nobody if the slot was its last user (and may be rebuilt for the new constants below).  Other stream
    // groups keep running on their own variants, which assign() never touches while a slot uses them.
    cudaStream_t st = stream_of(h, slot);
    GG_CUDA(cudaStreamSynchronize(st));
    gg::CfgConst kc;
    gg::derive_config(*cfg, kc);
    const gg::ConfigRegistry before = h->variants;
    bool build = false;
    const int id = h->variants.assign(slot, kc, &build);
    if (build) {
        // On failure the slot keeps its old configuration.  A new id gets its buffer before anything is written, so a
        // failed allocation changes nothing.
        if ((rc = ensure_variant_buffer(h, id))) {
            h->variants = before;
            return rc;
        }
        if ((rc = build_variant(h, id, st))) {
            // A launch error leaves the table untouched; an unused id whose table may have been partly rewritten no
            // longer holds the data of its old constants.  (A fault inside the kernel leaves the CUDA context failing
            // every later call, the slot's own old variant included.)
            h->variants = before;
            if (id < before.ids() && before.refs(id) == 0) h->variants.invalidate(id);
            return rc;
        }
    }
    h->slot_cfg[slot] = *cfg;
    return GG_OK;
}

int gg_get_slot_config(gg_handle h, int slot, gg_config* cfg) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!cfg) return fail(GG_E_ARG, "null argument");
    *cfg = h->slot_cfg[slot];
    return GG_OK;
}

int gg_init_map(gg_handle h, int slot, double x, double y, double z) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if ((rc = take_position_back(h, slot))) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    SlotState& s = h->slots[slot];
    s = SlotState();
    s.px = x;
    s.py = y;
    s.have_map = true;
    h->launches += gg::launch_init_map(h->view, slot, (float)z, stream_of(h, slot));
    GG_CUDA(cudaGetLastError());
    return GG_OK;
}

int gg_update_pose_batch(gg_handle h, int count, const int* slots, const double* xy, const double* T, int* moved) {
    if (!h || !slots || !xy || !T) return fail(GG_E_ARG, "null argument");
    if (count <= 0) return GG_OK;
    int rc;
    if ((rc = check_slots(h, count, slots))) return rc;
    for (int i = 0; i < count; ++i)
        if ((rc = take_position_back(h, slots[i]))) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    auto fill = [&](int i, Staging& e) {
        SlotState& s = h->slots[slots[i]];
        gg::SlotParams& p = e.hp[e.m];
        std::memset(&p, 0, sizeof(p));
        gg::move_map(h->view.k.res, s.px, s.py, xy[2 * i], xy[2 * i + 1], p.shift_i, p.shift_j);
        p.px = s.px;
        p.py = s.py;
        const double* t = T + 12 * (size_t)i;
        p.t20 = t[8];
        p.t21 = t[9];
        p.t22 = t[10];
        p.t23 = t[11];
        p.slot = slots[i];
        const bool mv = p.shift_i != 0 || p.shift_j != 0;   // else: "We havent moved so we have nothing to do", GroundGrid.cpp:136-137
        if (moved) moved[i] = mv ? 1 : 0;
        if (mv) s.moved_since_scan = true;
        return mv;
    };
    return run_groups(h, count, slots, false, nullptr, fill,
                      [&](const Staging& e, cudaStream_t st) { return gg::launch_roll(h->view, e.dp, e.m, st, h->prof); });
}

int gg_update_pose(gg_handle h, int slot, double x, double y, const double T[12], int* moved) {
    const double xy[2] = {x, y};
    return gg_update_pose_batch(h, 1, &slot, xy, T, moved);
}

int gg_get_map_position(gg_handle h, int slot, double xy[2]) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!xy) return fail(GG_E_ARG, "null argument");
    if ((rc = take_position_back(h, slot))) return rc;
    xy[0] = h->slots[slot].px;
    xy[1] = h->slots[slot].py;
    return GG_OK;
}

int gg_set_map_position(gg_handle h, int slot, double x, double y) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if ((rc = take_position_back(h, slot))) return rc;
    h->slots[slot].px = x;
    h->slots[slot].py = y;
    return GG_OK;
}

int gg_upload_points(gg_handle h, int slot, const gg_point* points, size_t n) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (n > h->pcap) return fail(GG_E_ARG, "%zu points exceed capacity %zu", n, h->pcap);
    if (n && !points) return fail(GG_E_ARG, "null points");
    h->inputs_busy = true;
    GG_CUDA(cudaSetDevice(h->device));
    if (n) GG_CUDA(cudaMemcpyAsync(h->view.points + (size_t)slot * h->pcap, points, n * sizeof(gg_point), cudaMemcpyHostToDevice, stream_of(h, slot)));
    h->slots[slot].n_points = n;
    return GG_OK;
}

int gg_run_scans(gg_handle h, int count, const gg_scan_desc* scans, int stop_after) {
    if (!h || !scans) return fail(GG_E_ARG, "null argument");
    if (stop_after < 0 || stop_after > 3) return fail(GG_E_ARG, "stop_after must be 0..3");
    h->inputs_busy = true;
    GG_CUDA(cudaSetDevice(h->device));
    return run_scans_grouped(h, count, scans, stop_after);
}

int gg_run_scans_device(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* dev_points, int stop_after) {
    if (!h || !scans || !dev_points) return fail(GG_E_ARG, "null argument");
    if (stop_after < 0 || stop_after > 3) return fail(GG_E_ARG, "stop_after must be 0..3");
    h->inputs_busy = true;
    for (int i = 0; i < count; ++i)
        if (!dev_points[i] && scans[i].n_points) return fail(GG_E_ARG, "scan %d: null device cloud", i);
    GG_CUDA(cudaSetDevice(h->device));
    return run_scans_grouped(h, count, scans, stop_after, dev_points);
}

namespace {
bool ranges_overlap(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
    const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return a && b && a_bytes && b_bytes && x < y + b_bytes && y < x + a_bytes;
}

// The output rules of gg_run_scans_to_device and gg_run_cloud_msgs_to_device: for the call, known select bits and an
// aligned dev_counts (scan < 0); for scan i, index / cloud only with select bits and dev_counts, each aligned.
int check_outputs(const gg_scan_outputs* outs, int scan, unsigned select, const int32_t* dev_counts) {
    if (scan < 0) {
        if (select & ~(GG_SELECT_GROUND | GG_SELECT_NONGROUND)) return fail(GG_E_ARG, "unknown select bits 0x%x", select);
        if (reinterpret_cast<uintptr_t>(dev_counts) % alignof(int32_t)) return fail(GG_E_ARG, "dev_counts is not 4-byte aligned");
        return GG_OK;
    }
    if (!outs) return GG_OK;
    const gg_scan_outputs& o = outs[scan];
    if (o.index || o.cloud) {
        if (!select) return fail(GG_E_ARG, "scan %d: index / cloud requested with select 0", scan);
        if (!dev_counts) return fail(GG_E_ARG, "scan %d: index / cloud requested without dev_counts", scan);
    }
    if (reinterpret_cast<uintptr_t>(o.index) % 4) return fail(GG_E_ARG, "scan %d: index is not 4-byte aligned", scan);
    if (reinterpret_cast<uintptr_t>(o.cloud) % 16) return fail(GG_E_ARG, "scan %d: cloud is not 16-byte aligned", scan);
    return GG_OK;
}
}  // namespace

int gg_run_scans_to_device(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* dev_points, const gg_scan_outputs* outs,
                           unsigned select, int32_t* dev_counts, void* stream) {
    if (!h || !scans || !dev_points) return fail(GG_E_ARG, "null argument");
    int rc;
    if ((rc = check_outputs(outs, -1, select, dev_counts))) return rc;
    h->inputs_busy = true;
    for (int i = 0; i < count; ++i) {
        const size_t n = scans[i].n_points;
        const gg_point* in = dev_points[i];
        if (!in && n) return fail(GG_E_ARG, "scan %d: null device cloud", i);
        if (ranges_overlap(dev_counts ? dev_counts + i : nullptr, sizeof(int32_t), in, n * sizeof(gg_point)))
            return fail(GG_E_ARG, "scan %d: dev_counts overlaps the input cloud", i);
        if ((rc = check_outputs(outs, i, select, dev_counts))) return rc;
        if (!outs) continue;
        const gg_scan_outputs& o = outs[i];
        if (ranges_overlap(o.labels, n, in, n * sizeof(gg_point)) || ranges_overlap(o.index, n * sizeof(uint32_t), in, n * sizeof(gg_point)) ||
            ranges_overlap(o.cloud, n * sizeof(gg_point), in, n * sizeof(gg_point)))
            return fail(GG_E_ARG, "scan %d: an output overlaps the input cloud", i);
    }
    GG_CUDA(cudaSetDevice(h->device));
    const CallerOutputs caller{outs, select, dev_counts, static_cast<cudaStream_t>(stream)};
    return run_scans_grouped(h, count, scans, 0, dev_points, nullptr, nullptr, &caller);
}

// ---- "next" rows of SURVEY.md section 8(f) --------------------------------------------------
namespace {
// gg_upload_cloud_msg[s] after validation: the host payloads are copied back to back into the slot's stream-group
// buffer d_raw (grown to their total bytes), then each part is a one-scan batch of the unpack kernel of
// gg_run_cloud_msgs_to_device, landing after the parts before it.
int upload_parts(gg_handle h, int slot, int n_parts, const gg_cloud_part* parts) {
    GG_CUDA(cudaSetDevice(h->device));
    h->inputs_busy = true;
    cudaStream_t st = stream_of(h, slot);
    const int sg = stream_index(h, slot);
    size_t bytes = 0, n_points = 0;
    for (int p = 0; p < n_parts; ++p) bytes += parts[p].n_points * (size_t)parts[p].msg.point_step;
    if (bytes > h->d_raw_cap[sg]) {
        GG_CUDA(cudaStreamSynchronize(st));   // the only users of this buffer are on `st`
        if (h->d_raw[sg]) GG_CUDA(cudaFree(h->d_raw[sg]));
        h->d_raw[sg] = nullptr;
        h->d_raw_cap[sg] = 0;
        GG_CUDA(cudaMalloc(reinterpret_cast<void**>(&h->d_raw[sg]), bytes + 256));
        h->d_raw_cap[sg] = bytes;
    }
    int rc;
    size_t at = 0;
    for (int p = 0; p < n_parts; ++p) {
        const gg_cloud_part& part = parts[p];
        const size_t part_bytes = part.n_points * (size_t)part.msg.point_step;
        if (part_bytes) GG_CUDA(cudaMemcpyAsync(h->d_raw[sg] + at, part.msg.data, part_bytes, cudaMemcpyHostToDevice, st));
        auto fill = [&](int, Staging& e) {
            std::memset(&e.hp[0], 0, sizeof(gg::SlotParams));
            e.hp[0].slot = slot;
            e.hp[0].n_points = (int)part.n_points;
            fill_unpack(e.hunpack[0], h->d_raw[sg] + at, part.msg.point_step, part.msg.field_offsets, part.msg.T_map_from_frame);
            e.hunpack[0].first = (int)n_points;
            e.unpack = true;
            return true;
        };
        auto launch = [&](const Staging& e, cudaStream_t s) { return gg::launch_unpack(h->view, e.dp, e.dunpack, 1, e.max_points, s, h->prof); };
        if ((rc = run_groups(h, 1, &slot, false, nullptr, fill, launch))) return rc;
        at += part_bytes;
        n_points += part.n_points;
    }
    h->slots[slot].n_points = n_points;
    return GG_OK;
}
}  // namespace

int gg_upload_cloud_msg(gg_handle h, int slot, const void* data, size_t n_points, int point_step, const int field_offsets[5],
                        const double T_map_from_frame[12]) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (n_points > h->pcap) return fail(GG_E_ARG, "%zu points exceed capacity %zu", n_points, h->pcap);
    if ((rc = check_cloud_msg(data, n_points, point_step, field_offsets))) return rc;
    gg_cloud_part part{{data, point_step, {}, T_map_from_frame}, n_points};
    std::memcpy(part.msg.field_offsets, field_offsets, sizeof(part.msg.field_offsets));
    return upload_parts(h, slot, 1, &part);
}

int gg_upload_cloud_msgs(gg_handle h, int slot, int n_parts, const gg_cloud_part* parts) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (n_parts < 0 || n_parts > GG_MAX_CLOUD_PARTS) return fail(GG_E_ARG, "%d parts, not in [0, %d]", n_parts, GG_MAX_CLOUD_PARTS);
    if (n_parts && !parts) return fail(GG_E_ARG, "null parts");
    size_t n_points = 0;
    for (int p = 0; p < n_parts; ++p) {
        const gg_cloud_part& part = parts[p];
        if ((rc = check_cloud_msg(part.msg.data, part.n_points, part.msg.point_step, part.msg.field_offsets)))
            return fail(rc, "part %d: %s", p, g_last_error.c_str());
        if (part.n_points > h->pcap - n_points) return fail(GG_E_ARG, "part %d: the parts exceed capacity %zu", p, h->pcap);
        n_points += part.n_points;
    }
    return upload_parts(h, slot, n_parts, parts);
}

int gg_run_cloud_msgs_to_device(gg_handle h, int count, const gg_scan_desc* scans, const gg_cloud_msg* msgs, const gg_scan_outputs* outs,
                                unsigned select, int32_t* dev_counts, void* stream) {
    if (!h || !scans || !msgs) return fail(GG_E_ARG, "null argument");
    int rc;
    if ((rc = check_outputs(outs, -1, select, dev_counts))) return rc;
    for (int i = 0; i < count; ++i) {
        const gg_cloud_msg& m = msgs[i];
        if ((rc = check_cloud_msg(m.data, scans[i].n_points, m.point_step, m.field_offsets))) return fail(rc, "scan %d: %s", i, g_last_error.c_str());
        // outputs may overlap the scan's own payload: the output kernels read the slot's buffer, and the payload has
        // been consumed by the unpack kernel that runs before them on the same stream
        if ((rc = check_outputs(outs, i, select, dev_counts))) return rc;
    }
    h->inputs_busy = true;
    GG_CUDA(cudaSetDevice(h->device));
    const CallerOutputs caller{outs, select, dev_counts, static_cast<cudaStream_t>(stream), msgs};
    return run_scans_grouped(h, count, scans, 0, nullptr, nullptr, nullptr, &caller);
}

int gg_run_merged_cloud_msgs_to_device(gg_handle h, int count, const gg_scan_desc* scans, const int* n_parts, const gg_cloud_part* parts,
                                       const gg_scan_outputs* outs, unsigned select, int32_t* dev_counts, void* stream) {
    if (!h || !scans || (count > 0 && (!n_parts || !parts))) return fail(GG_E_ARG, "null argument");
    int rc;
    if ((rc = check_outputs(outs, -1, select, dev_counts))) return rc;
    std::vector<int>& base = h->part_base;
    base.assign((size_t)std::max(count, 0), 0);
    int next = 0;
    for (int i = 0; i < count; ++i) {
        const int m = n_parts[i];
        if (m < 0 || m > GG_MAX_CLOUD_PARTS) return fail(GG_E_ARG, "scan %d: %d parts, not in [0, %d]", i, m, GG_MAX_CLOUD_PARTS);
        base[i] = next;
        size_t n = 0;
        for (int p = 0; p < m; ++p) {
            const gg_cloud_part& part = parts[next + p];
            if ((rc = check_cloud_msg(part.msg.data, part.n_points, part.msg.point_step, part.msg.field_offsets)))
                return fail(rc, "scan %d part %d: %s", i, p, g_last_error.c_str());
            if (part.n_points > scans[i].n_points - n)
                return fail(GG_E_ARG, "scan %d: its parts hold more than its n_points %zu", i, scans[i].n_points);
            n += part.n_points;
        }
        if (n != scans[i].n_points) return fail(GG_E_ARG, "scan %d: its parts hold %zu points, its n_points is %zu", i, n, scans[i].n_points);
        next += m;
        // as in gg_run_cloud_msgs_to_device, outputs may overlap the scan's own parts: every part is consumed before the
        // scan's first kernel on the same stream
        if ((rc = check_outputs(outs, i, select, dev_counts))) return rc;
    }
    h->inputs_busy = true;
    GG_CUDA(cudaSetDevice(h->device));
    CallerOutputs caller{outs, select, dev_counts, static_cast<cudaStream_t>(stream), nullptr};
    caller.n_parts = n_parts;
    caller.parts = parts;
    caller.part_base = base.data();
    return run_scans_grouped(h, count, scans, 0, nullptr, nullptr, nullptr, &caller);
}

namespace {
// A caller-owned device buffer of a batched slot call.
struct CallerBuf {
    const void* p;
    size_t bytes;
    size_t align;
    bool required;     // false: may be null
    const char* what;
};

// The validation shared by the batched calls on a set of slots and layer names (gg_get_layers_to_device,
// gg_set_layers_from_device, gg_layer_images_to_device, gg_terrain_images_to_device), in this order: the handle, the
// counts (count == 0 or n_names == 0 is a valid call with nothing to do: GG_OK, and the caller enqueues nothing), null
// arguments, at most L_NUM names, each buffer (aligned, outside the layer arena, disjoint from the other buffers),
// the slot checks of check_slots, `n_names` distinct names resolved as gg_get_layer
// resolves them ("points" per slot, as LAYER_POINTS at *points_at; "expectedPoints" is not a layer of a slot).
// A call without layer names (gg_eval_counts_to_device) passes list == nullptr: n_names and names are then ignored.
int check_slot_batch(gg_handle h, int count, const int* slots, int n_names, const char* const* names, std::initializer_list<CallerBuf> bufs,
                     gg::LayerList* list, int* points_at) {
    const bool named = list != nullptr;
    if (!h) return fail(GG_E_ARG, "null handle");
    if (count < 0 || (named && n_names < 0)) return fail(GG_E_ARG, "negative count");
    if (count == 0 || (named && n_names == 0)) return GG_OK;
    if (!slots || (named && !names)) return fail(GG_E_ARG, "null argument");
    for (const CallerBuf& b : bufs)
        if (b.required && !b.p) return fail(GG_E_ARG, "null argument");
    if (named && n_names > gg::L_NUM) return fail(GG_E_ARG, "%d layer names, at most %d", n_names, (int)gg::L_NUM);
    const gg::View& v = h->view;
    const size_t arena = (size_t)h->n_slots * v.n_layers * v.k.N2 * sizeof(float);
    for (const CallerBuf& b : bufs) {
        if (!b.p) continue;
        if (reinterpret_cast<uintptr_t>(b.p) % b.align) return fail(GG_E_ARG, "%s is not %zu-byte aligned", b.what, b.align);
        if (ranges_overlap(b.p, b.bytes, v.layers, arena)) return fail(GG_E_ARG, "%s overlaps the handle's layers", b.what);
        for (const CallerBuf& o : bufs)
            if (&o < &b && o.p && ranges_overlap(b.p, b.bytes, o.p, o.bytes)) return fail(GG_E_ARG, "%s overlaps %s", b.what, o.what);
    }
    int rc;
    if ((rc = check_slots(h, count, slots))) return rc;
    if (!named) return GG_OK;
    list->n = n_names;
    for (int l = 0; l < n_names; ++l) {
        const char* name = names[l];
        if (!name) return fail(GG_E_ARG, "null layer name");
        for (int m = 0; m < l; ++m)
            if (std::strcmp(names[m], name) == 0) return fail(GG_E_ARG, "layer '%s' appears twice", name);
        if (std::strcmp(name, "expectedPoints") == 0) return fail(GG_E_LAYER, "'expectedPoints' is a table of the handle, not a layer of a slot");
        if (std::strcmp(name, "points") == 0) {
            list->idx[l] = gg::LAYER_POINTS;
            *points_at = l;
        } else if ((rc = layer_index(h, slots[0], name, &list->idx[l]))) {
            return rc;
        }
    }
    return GG_OK;
}

// Per-block range scratch of the layer images (launch_layer_images), allocated on first use.
int ensure_image_partials(gg_handle h) {
    if (h->d_img_part) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    const size_t n = (size_t)h->n_slots * gg::L_NUM * ((h->view.k.N2 + gg::IMG_RANGE_CELLS - 1) / gg::IMG_RANGE_CELLS);
    return dev_alloc(h, &h->d_img_part, n);
}

int layer_images(gg_handle h, int count, const int* slots, const gg::LayerList& list, uint8_t* dst, float* dev_range, void* stream) {
    return enqueue_slot_batch(h, count, slots, stream, [&](const Staging& e, cudaStream_t st) {
        return gg::launch_layer_images(h->view, e.dp, e.m, list, h->d_img_part, dst, dev_range, st, h->prof);
    });
}

int terrain_images(gg_handle h, int count, const int* slots, float* dst, void* stream) {
    return enqueue_slot_batch(h, count, slots, stream, [&](const Staging& e, cudaStream_t st) {
        return gg::launch_terrain_images(h->view, e.dp, e.m, dst, st, h->prof);
    });
}

// f4: the rule of every evaluation call (the scan's labels are complete)
int check_completed_scan(gg_handle h, int slot) {
    const SlotState& s = h->slots[slot];
    if (!s.ran || s.last_stop != 0) return fail(GG_E_STATE, "slot %d: no completed scan", slot);
    return GG_OK;
}

// per slot its last scan's input (n_points, src / packed as the scan saw them) and its position in the call
int eval_counts(gg_handle h, int count, const int* slots, unsigned long long* dst, void* stream) {
    GG_CUDA(cudaSetDevice(h->device));
    int max_points = 0;
    for (int i = 0; i < count; ++i) max_points = std::max(max_points, (int)h->slots[slots[i]].n_points);
    auto fill = [&](int i, Staging& e) {
        const SlotState& s = h->slots[slots[i]];
        gg::SlotParams& p = e.hp[e.m];
        std::memset(&p, 0, sizeof(p));
        p.slot = slots[i];
        p.pos = i;
        p.n_points = (int)s.n_points;
        p.src = s.src ? s.src : h->view.points + (size_t)slots[i] * h->pcap;
        p.packed = s.packed_input;
        return true;
    };
    auto launch = [&](const Staging& e, cudaStream_t st) { return gg::launch_eval(h->view, e.dp, e.m, max_points, dst, st, h->prof); };
    return run_groups(h, count, slots, true, static_cast<cudaStream_t>(stream), fill, launch);
}
}  // namespace

// f3: the per-slot calls are one-scan batches of the kernels of gg_terrain_images_to_device / gg_layer_images_to_device
// on the slot's own stream, followed by a pageable copy and a synchronise.
int gg_terrain_image(gg_handle h, int slot, float* dst) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!dst) return fail(GG_E_ARG, "null dst");
    if (!(h->flags & GG_FLAG_FULL_LAYERS)) return fail(GG_E_LAYER, "the terrain image needs 'pointsRaw' (GG_FLAG_FULL_LAYERS)");
    GG_CUDA(cudaSetDevice(h->device));
    const size_t n = (size_t)h->view.k.N2 * 3;
    if (!h->d_image && (rc = dev_alloc(h, &h->d_image, n))) return rc;
    cudaStream_t st = stream_of(h, slot);
    if ((rc = terrain_images(h, 1, &slot, h->d_image, st))) return rc;
    GG_CUDA(cudaMemcpyAsync(dst, h->d_image, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaStreamSynchronize(st));
    return GG_OK;
}

// f3: the single-channel 8-bit image cv::applyColorMap receives (GroundGridNodelet.cpp:238-245)
int gg_layer_image_u8(gg_handle h, int slot, const char* name, uint8_t* dst, float* lower, float* upper) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!name || !dst) return fail(GG_E_ARG, "null argument");
    gg::LayerList list{};
    list.n = 1;
    if ((rc = layer_index(h, slot, name, &list.idx[0]))) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    const size_t n = (size_t)h->view.k.N2;
    if (!h->d_image_u8) {
        if ((rc = dev_alloc(h, &h->d_image_u8, n))) return rc;
        if ((rc = dev_alloc(h, &h->d_minmax, 2))) return rc;
    }
    if ((rc = ensure_image_partials(h))) return rc;
    cudaStream_t st = stream_of(h, slot);
    if ((rc = layer_images(h, 1, &slot, list, h->d_image_u8, h->d_minmax, st))) return rc;
    float range[2];
    GG_CUDA(cudaMemcpyAsync(dst, h->d_image_u8, n, cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaMemcpyAsync(range, h->d_minmax, sizeof(range), cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaStreamSynchronize(st));
    if (lower) *lower = range[0];
    if (upper) *upper = range[1];
    return GG_OK;
}

int gg_layer_images_to_device(gg_handle h, int count, const int* slots, int n_names, const char* const* names, uint8_t* dst, float* dev_range,
                              void* stream) {
    gg::LayerList list{};
    int points_at = -1, rc;
    const size_t planes = (size_t)count * n_names, plane = h ? (size_t)h->view.k.N2 : 0;
    if ((rc = check_slot_batch(h, count, slots, n_names, names,
                               {{dst, planes * plane, 1, true, "dst"}, {dev_range, planes * 2 * sizeof(float), alignof(float), false, "dev_range"}},
                               &list, &points_at)) ||
        count == 0 || n_names == 0)
        return rc;
    if ((rc = ensure_image_partials(h))) return rc;
    return layer_images(h, count, slots, list, dst, dev_range, stream);
}

int gg_terrain_images_to_device(gg_handle h, int count, const int* slots, float* dst, void* stream) {
    // the terrain image reads "pointsRaw": resolving that name rejects a handle without the full layers (GG_E_LAYER)
    static const char* const raw[1] = {"pointsRaw"};
    gg::LayerList list{};
    int points_at = -1, rc;
    const size_t bytes = h ? (size_t)count * h->view.k.N2 * 3 * sizeof(float) : 0;
    if ((rc = check_slot_batch(h, count, slots, 1, raw, {{dst, bytes, alignof(float), true, "dst"}}, &list, &points_at)) || count == 0)
        return rc;
    return terrain_images(h, count, slots, dst, stream);
}

// ---- single phases (GroundSegmentation.h:56-62 of the reference) ------------------------------
// Both read the plane "points" names (layer_index); the whole-map call first recomputes the variance from "m2" (:323)
// where the handle keeps it (GG_FLAG_FULL_LAYERS), else it reads the stored variance.
int gg_detect_ground_patches(gg_handle h, int slot) {
    int rc = check_slot(h, slot), points = gg::L_COUNT;
    if (rc || (rc = layer_index(h, slot, "points", &points))) return rc;
    const bool recompute = (h->flags & GG_FLAG_FULL_LAYERS) != 0;
    return run_phase(h, slot, 0.0, [&](const Staging& e, cudaStream_t st) {
        return gg::launch_detect_only(h->view, e.dp, 1, st, h->prof, h->have_layer_map ? &h->layer_map : nullptr, points, recompute);
    });
}

int gg_spiral_ground_interpolation(gg_handle h, int slot, double base_z) {
    return run_phase(h, slot, base_z, [&](const Staging& e, cudaStream_t st) { return gg::launch_spiral_only(h->view, e.dp, 1, st, h->prof); });
}

int gg_interpolate_cell(gg_handle h, int slot, int x, int y) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    const int N = h->view.k.N;
    if (x < 1 || y < 1 || x >= N - 1 || y >= N - 1) return fail(GG_E_ARG, "cell (%d, %d) has no 3x3 neighbourhood", x, y);
    GG_CUDA(cudaSetDevice(h->device));
    h->launches += gg::launch_interpolate_cell(h->view, h->variants.constants(h->variants.variant_of(slot)), slot, x, y, stream_of(h, slot));
    GG_CUDA(cudaGetLastError());
    return GG_OK;
}

int gg_detect_ground_patch(gg_handle h, int slot, int patch_size, int i, int j) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (patch_size != 3 && patch_size != 5) return fail(GG_E_ARG, "patch size must be 3 or 5");
    const int N = h->view.k.N, H = patch_size / 2;
    if (i < H || j < H || i >= N - H || j >= N - H) return fail(GG_E_ARG, "cell (%d, %d) has no %dx%d neighbourhood", i, j, patch_size, patch_size);
    int points = gg::L_COUNT;
    if ((rc = layer_index(h, slot, "points", &points))) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    h->launches += gg::launch_detect_cell(h->view, h->variants.constants(h->variants.variant_of(slot)), slot, patch_size, i, j, points,
                                          stream_of(h, slot));
    GG_CUDA(cudaGetLastError());
    return GG_OK;
}

// class << 24 | cell of every input point of the slot's last rasterisation (the index lists insert_cloud fills)
int gg_get_point_classes(gg_handle h, int slot, uint32_t* codes, size_t n) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (n > h->slots[slot].n_points || (n && !codes)) return fail(GG_E_ARG, "bad class buffer");
    if (!h->slots[slot].ran) return fail(GG_E_STATE, "slot %d: no rasterised scan", slot);
    GG_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream_of(h, slot);
    if (n) GG_CUDA(cudaMemcpyAsync(codes, h->view.code + (size_t)slot * h->pcap, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaStreamSynchronize(st));
    return GG_OK;
}

// f4: a one-scan batch of gg_eval_counts_to_device into the handle's tally, on the slot's own stream
int gg_eval_accumulate(gg_handle h, int slot) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if ((rc = check_completed_scan(h, slot))) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    if (!h->d_eval) {
        if ((rc = dev_alloc(h, &h->d_eval, (size_t)gg::EVAL_LABELS * 2))) return rc;
        GG_CUDA(cudaMemset(h->d_eval, 0, sizeof(unsigned long long) * gg::EVAL_LABELS * 2));
    }
    return eval_counts(h, 1, &slot, h->d_eval, stream_of(h, slot));
}

int gg_eval_counts_to_device(gg_handle h, int count, const int* slots, uint64_t* dev_counts, void* stream) {
    static_assert(sizeof(uint64_t) == sizeof(unsigned long long), "64-bit tallies");
    int rc;
    const size_t bytes = count > 0 ? (size_t)count * gg::EVAL_LABELS * 2 * sizeof(uint64_t) : 0;
    if ((rc = check_slot_batch(h, count, slots, 0, nullptr, {{dev_counts, bytes, alignof(uint64_t), true, "dev_counts"}}, nullptr, nullptr)) ||
        count == 0)
        return rc;
    for (int i = 0; i < count; ++i)
        if ((rc = check_completed_scan(h, slots[i]))) return rc;
    return eval_counts(h, count, slots, reinterpret_cast<unsigned long long*>(dev_counts), stream);
}

int gg_eval_read(gg_handle h, uint64_t* counts, int reset) {
    if (!h || !counts) return fail(GG_E_ARG, "null argument");
    int rc = gg_synchronize(h);
    if (rc) return rc;
    const size_t bytes = sizeof(unsigned long long) * gg::EVAL_LABELS * 2;
    if (!h->d_eval) {
        std::memset(counts, 0, bytes);
        return GG_OK;
    }
    GG_CUDA(cudaMemcpy(counts, h->d_eval, bytes, cudaMemcpyDeviceToHost));
    if (reset) GG_CUDA(cudaMemset(h->d_eval, 0, bytes));
    return GG_OK;
}

int gg_profile_enable(gg_handle h, int on) {
    if (!h) return fail(GG_E_ARG, "null handle");
    GG_CUDA(cudaSetDevice(h->device));
    if (on && !h->prof) h->prof = new EventProfiler();
    if (!on && h->prof) {
        int rc = gg_synchronize(h);
        if (rc) return rc;
        h->prof->collect(h->prof_ms, h->prof_count);
        delete h->prof;
        h->prof = nullptr;
    }
    return GG_OK;
}

int gg_profile_read(gg_handle h, double* ms_per_kernel, uint32_t* launches_per_kernel, int reset) {
    if (!h) return fail(GG_E_ARG, "null handle");
    int rc = gg_synchronize(h);
    if (rc) return rc;
    if (h->prof) h->prof->collect(h->prof_ms, h->prof_count);
    for (int k = 0; k < gg::K_NUM; ++k) {
        if (ms_per_kernel) ms_per_kernel[k] = h->prof_ms[k];
        if (launches_per_kernel) launches_per_kernel[k] = h->prof_count[k];
        if (reset) {
            h->prof_ms[k] = 0.0;
            h->prof_count[k] = 0;
        }
    }
    return GG_OK;
}

int gg_profile_kernel_count(void) { return gg::K_NUM; }

const char* gg_profile_kernel_name(int id) {
    static const char* names[gg::K_NUM] = {"k_rasterize",   "k_cell_tiles",    "k_cell_place",    "k_scatter",
                                           "k_cell_stats",  "k_detect",        "k_spiral",           "k_label",         "k_roll_gather",
                                           "k_roll_commit", "k_out_count",     "k_out_scan",         "k_out_write",     "k_unpack_transform",
                                           "k_terrain_image", "k_eval_counts", "k_layer_copy", "k_layer_range", "k_layer_image",
                                           "k_sample_layers", "k_point_info", "k_stage_poses", "k_pose_resolve"};
    return (id >= 0 && id < gg::K_NUM) ? names[id] : "";
}

int gg_download_labels(gg_handle h, int slot, uint8_t* labels_out, size_t n) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (n > h->pcap || (n && !labels_out)) return fail(GG_E_ARG, "bad label buffer");
    GG_CUDA(cudaSetDevice(h->device));
    if (n) GG_CUDA(cudaMemcpyAsync(labels_out, h->view.labels + (size_t)slot * h->pcap, n, cudaMemcpyDeviceToHost, stream_of(h, slot)));
    return GG_OK;
}

int gg_synchronize(gg_handle h) {
    if (!h) return fail(GG_E_ARG, "null handle");
    GG_CUDA(cudaSetDevice(h->device));
    for (int i = 0; i < h->n_streams; ++i) GG_CUDA(cudaStreamSynchronize(h->streams[i]));
    if (h->copy_out) GG_CUDA(cudaStreamSynchronize(h->copy_out));
    h->batch_outstanding[0] = h->batch_outstanding[1] = false;
    h->inputs_busy = false;
    return GG_OK;
}

int gg_get_output(gg_handle h, int slot, uint32_t* index_out, gg_point* cloud_out, size_t* n_out) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = stream_of(h, slot);
    if ((rc = run_output_on(h, slot, cloud_out != nullptr))) return rc;
    int total = 0;
    const gg::View& v = h->view;
    GG_CUDA(cudaMemcpyAsync(&total, v.out_counts + (size_t)slot * (3 * v.out_blocks + 1) + 3 * v.out_blocks, sizeof(int), cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaStreamSynchronize(st));
    if (n_out) *n_out = (size_t)total;
    if (index_out && total) GG_CUDA(cudaMemcpyAsync(index_out, v.out_index + (size_t)slot * h->pcap, (size_t)total * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    if (cloud_out && total) GG_CUDA(cudaMemcpyAsync(cloud_out, v.out_cloud + (size_t)slot * h->pcap, (size_t)total * sizeof(gg_point), cudaMemcpyDeviceToHost, st));
    GG_CUDA(cudaStreamSynchronize(st));
    return GG_OK;
}

int gg_filter_cloud(gg_handle h, int slot, const gg_point* points, size_t n, const float origin[3], double base_z,
                    uint8_t* labels_out, uint32_t* index_out, gg_point* cloud_out, size_t* n_out) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!origin) return fail(GG_E_ARG, "null origin");
    if (!h->slots[slot].have_map) return fail(GG_E_STATE, "slot %d: map not initialised", slot);
    if ((rc = gg_upload_points(h, slot, points, n))) return rc;
    gg_scan_desc d;
    std::memset(&d, 0, sizeof(d));
    d.slot = slot;
    d.n_points = n;
    d.origin[0] = origin[0];
    d.origin[1] = origin[1];
    d.origin[2] = origin[2];
    d.base_z = base_z;
    if ((rc = run_scans_grouped(h, 1, &d, 0))) return rc;
    if (labels_out && (rc = gg_download_labels(h, slot, labels_out, n))) return rc;
    if (index_out || cloud_out || n_out) return gg_get_output(h, slot, index_out, cloud_out, n_out);
    GG_CUDA(cudaStreamSynchronize(stream_of(h, slot)));
    return GG_OK;
}

namespace {

int batch_wait(gg_handle h, int parity) {
    if (h->batch_outstanding[parity]) {
        GG_CUDA(cudaEventSynchronize(h->batch_done[parity]));
        h->batch_outstanding[parity] = false;
    }
    return GG_OK;
}

// streams, events and the second buffer set of the batch path
int batch_prepare(gg_handle h) {
    int rc;
    if (!h->copy_out) {
        for (int e = 0; e < 8; ++e) GG_CUDA(cudaEventCreateWithFlags(&h->raw_ev[e], cudaEventDisableTiming));
        for (int e = 0; e < 2; ++e) GG_CUDA(cudaEventCreateWithFlags(&h->batch_done[e], cudaEventDisableTiming));
        for (int e = 0; e < h->n_copy_in + 2; ++e) GG_CUDA(cudaStreamCreateWithFlags(&h->copy_in[e], cudaStreamNonBlocking));
        GG_CUDA(cudaStreamCreateWithFlags(&h->copy_out, cudaStreamNonBlocking));
        h->in_raw[0] = h->view.points;
        h->labels_buf[0] = h->view.labels;
    }
    if (h->host_pack && !h->h_stage) {
        if ((rc = dev_alloc(h, &h->in_raw[1], (size_t)h->n_slots * h->pcap))) return rc;
        if ((rc = dev_alloc(h, &h->labels_buf[1], (size_t)h->n_slots * h->pcap))) return rc;
        for (int e = 0; e < 2; ++e)
            if ((rc = dev_alloc(h, &h->in_packed[e], (size_t)h->n_slots * 14 * h->pcap))) return rc;
        if (const char* e = getenv("GG_PACK_RING")) h->pack_slots = std::min(256, std::max(2, atoi(e)));
        GG_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h->h_stage), (size_t)h->pack_slots * 14 * h->pcap, cudaHostAllocDefault));
        h->slot_ev.resize(h->pack_slots);
        for (cudaEvent_t& e : h->slot_ev) GG_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        h->packer->set_ring(h->h_stage, 14 * h->pcap, h->pack_slots);
    }
    return GG_OK;
}

}  // namespace

int gg_filter_cloud_batch_begin(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* points, uint8_t* const* labels_out,
                                int* ticket) {
    if (!h || !scans || !points) return fail(GG_E_ARG, "null argument");
    if (count < 0) return fail(GG_E_ARG, "negative count");
    int rc;
    if ((rc = check_slots(h, count, scans, points))) return rc;
    GG_CUDA(cudaSetDevice(h->device));
    if (h->host_pack && !h->packer) {
        // GG_HOST_THREADS forces a thread count; by default all usable CPUs (affinity, cgroup quota,
        // shared between the local ranks) but one
        int threads = 0;
        if (const char* e = getenv("GG_HOST_THREADS")) threads = atoi(e);
        if (threads <= 0) {
            int local = 1;
            if (const char* e = getenv("LOCAL_WORLD_SIZE")) local = std::max(1, atoi(e));
            threads = std::min(48, gg::usable_cpus() / local - 1);
        }
        if (threads < 1)
            h->host_pack = 0;
        else
            h->packer = new HostPacker(threads);
    }
    if ((rc = batch_prepare(h))) return rc;
    while ((int)h->batch_ev.size() < h->n_streams) {  // [0, n_streams): one event per compute stream
        cudaEvent_t ev;
        GG_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        h->batch_ev.push_back(ev);
    }
    const int par = h->host_pack ? h->batch_parity : 0;
    // the batch that used this buffer set two calls ago must be complete (it normally is, long since)
    if ((rc = batch_wait(h, par))) return rc;
    h->last_raw = h->last_packed = h->last_raw_bytes = h->last_packed_bytes = 0;
    const auto t_begin = std::chrono::steady_clock::now();
    auto us_since = [&] { return (size_t)std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_begin).count(); };
    if (h->host_pack) {
        // Two ways to get a cloud across PCIe: repacked by host worker threads into x | y | z | ring
        // (14 useful bytes of every 32-byte record, costs CPU time) or as it is (costs bus time).  Both
        // resources are used at once: the packers walk the scans from the front; whenever fewer than
        // raw_depth raw copies of this loop are pending, the calling thread takes the LAST scan nobody has
        // started packing and sends it raw.  Whatever the CPU quota of the host, neither the packers
        // nor the bus sit idle.
        //
        // All clouds go through a few copy streams and all labels come back through another one, so a
        // transfer never queues behind kernels.  Events hand the scans over: copies -> kernels (the
        // stream of the slot) -> label read-back.  Kernels are enqueued for `launch_unit` delivered scans
        // of a stream group at a time, so that only the kernels of the last few scans run after the
        // transfers have ended.
        unsigned char* const dpk = h->in_packed[par];
        gg_point* const draw = h->in_raw[par];
        uint8_t* const dlab = h->labels_buf[par];
        h->view.labels = dlab;  // what gg_download_labels / gg_get_output read after this batch
        const int KP = h->n_copy_in, KC = KP + 2;  // packed clouds rotate over the first KP copy streams, raw ones over the last 2
        std::vector<int> order;
        for (int g = 0; g < h->n_streams; ++g)
            for (int i = 0; i < count; ++i)
                if (stream_index(h, scans[i].slot) == g) order.push_back(i);
        std::vector<PackJob> jobs(count);
        for (int k = 0; k < count; ++k) {
            const gg_scan_desc& d = scans[order[k]];
            jobs[k].src = points[order[k]];
            jobs[k].n = d.n_points;
        }
        if (h->inputs_busy) {  // earlier asynchronous calls may still use the slots' own input buffers
            for (int g = 0; g < h->n_streams; ++g) {
                GG_CUDA(cudaEventRecord(h->batch_ev[g], h->streams[g]));
                for (int c = 0; c < KC; ++c) GG_CUDA(cudaStreamWaitEvent(h->copy_in[c], h->batch_ev[g], 0));
            }
        }
        size_t ev_used = h->n_streams;
        auto next_event = [&](cudaEvent_t* ev) -> int {
            if (ev_used == h->batch_ev.size()) {
                cudaEvent_t e;
                GG_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
                h->batch_ev.push_back(e);
            }
            *ev = h->batch_ev[ev_used++];
            return GG_OK;
        };
        std::vector<std::vector<int>> pending(h->n_streams);  // delivered, kernels not yet enqueued (positions in `order`)
        std::vector<gg_scan_desc> ud;
        std::vector<const gg_point*> usrc;
        std::vector<const float*> upk;
        std::vector<unsigned char> sent_packed(count, 0);
        auto flush = [&](int g) -> int {
            std::vector<int>& pg = pending[g];
            if (pg.empty()) return GG_OK;
            ud.clear();
            usrc.clear();
            upk.clear();
            for (int k : pg) {
                const gg_scan_desc& d = scans[order[k]];
                ud.push_back(d);
                usrc.push_back(draw + (size_t)d.slot * h->pcap);
                upk.push_back(sent_packed[k] ? reinterpret_cast<const float*>(dpk + (size_t)d.slot * 14 * h->pcap) : nullptr);
            }
            cudaStream_t st = h->streams[g];
            cudaEvent_t ev;
            int rc2;
            for (int c = 0; c < KC; ++c) {  // the clouds are spread over all copy streams
                if ((rc2 = next_event(&ev))) return rc2;
                GG_CUDA(cudaEventRecord(ev, h->copy_in[c]));
                GG_CUDA(cudaStreamWaitEvent(st, ev, 0));
            }
            if ((rc2 = run_scans_grouped(h, (int)ud.size(), ud.data(), 0, usrc.data(), upk.data(), dlab))) return rc2;
            if (labels_out) {  // the labels travel under the remaining H2D traffic
                if ((rc2 = next_event(&ev))) return rc2;
                GG_CUDA(cudaEventRecord(ev, st));
                GG_CUDA(cudaStreamWaitEvent(h->copy_out, ev, 0));
                for (int k : pg)
                    if (labels_out[order[k]] && scans[order[k]].n_points)
                        GG_CUDA(cudaMemcpyAsync(labels_out[order[k]], dlab + (size_t)scans[order[k]].slot * h->pcap, scans[order[k]].n_points,
                                                cudaMemcpyDeviceToHost, h->copy_out));
            }
            pg.clear();
            return GG_OK;
        };
        auto delivered = [&](int k) -> int {
            const int g = stream_index(h, scans[order[k]].slot);
            pending[g].push_back(k);
            return (int)pending[g].size() >= h->launch_unit ? flush(g) : GG_OK;
        };
        const uint64_t seq_base = h->pack_issued;
        auto poll_copies = [&] {  // staging slots whose cloud has reached the device go back to the packers, in order
            uint64_t done = h->packer->copied.load(std::memory_order_relaxed);
            while (done < h->pack_issued && cudaEventQuery(h->slot_ev[done % (uint64_t)h->pack_slots]) == cudaSuccess) ++done;
            h->packer->copied.store(done, std::memory_order_release);
        };
        h->packer->pack_ns = 0;
        h->packer->slot_wait_ns = 0;
        uint64_t idle_ns = 0;
        h->packer->start(&jobs, seq_base);
        struct CancelOnExit {  // an error return below must not leave packers working on `jobs`
            HostPacker* p;
            bool armed = true;
            ~CancelOnExit() {
                if (armed) p->cancel();
            }
        } pack_guard{h->packer};
        int front = 0, back = count, raw_issued = 0, raw_done = 0, n_copies = 0;
        size_t last_packed_bytes = 14 * (size_t)h->pcap, last_raw_bytes = sizeof(gg_point) * (size_t)h->pcap;   // size of the latest copy of either kind
        while (front < back) {
            poll_copies();
            if (h->packer->packed(jobs[front])) {
                const gg_scan_desc& d = scans[order[front]];
                const size_t n_pad = (d.n_points + 7) & ~(size_t)7;
                cudaStream_t cs = h->copy_in[n_copies++ % KP];
                if (d.n_points)
                    GG_CUDA(cudaMemcpyAsync(dpk + (size_t)d.slot * 14 * h->pcap, h->packer->slot_of(h->pack_issued), 14 * n_pad, cudaMemcpyHostToDevice, cs));
                GG_CUDA(cudaEventRecord(h->slot_ev[h->pack_issued % (uint64_t)h->pack_slots], cs));
                ++h->pack_issued;
                sent_packed[front] = 1;
                ++h->last_packed;
                h->last_packed_bytes += 14 * n_pad;
                last_packed_bytes = 14 * n_pad;
                if ((rc = delivered(front))) return rc;
                ++front;
                continue;
            }
            // A raw cloud costs 32 B/point of bus time, a packed one 14, so packed clouds go first whenever one is ready.
            // What the packers cannot fill is topped up with raw clouds: the measure is the number of BYTES in flight on
            // the bus (copies issued and not yet completed, both kinds).  Below the target the DMA engines would run dry
            // before the next packed cloud arrives, so a raw one is added; above it the bus is the limit and a raw cloud
            // would only delay cheaper packed ones.  The split therefore follows the measured rates of the packers and of
            // the bus on this host (CPU quota, ranks sharing the socket) instead of a fixed gate.
            while (raw_done < raw_issued && cudaEventQuery(h->raw_ev[raw_done % h->raw_depth]) == cudaSuccess) ++raw_done;
            const uint64_t packed_in_flight = h->pack_issued - h->packer->copied.load(std::memory_order_relaxed);
            const size_t in_flight_bytes = (size_t)packed_in_flight * last_packed_bytes + (size_t)(raw_issued - raw_done) * last_raw_bytes;
            const bool below_target = h->bus_target ? in_flight_bytes < h->bus_target : packed_in_flight < (uint64_t)h->raw_gate;
            const bool bus_free = h->host_pack_mix && below_target && (raw_issued - raw_done) < h->raw_depth;
            int j = bus_free ? h->packer->claim_raw_from_back() : -1;
            if (j >= 0) {
                const gg_scan_desc& d = scans[order[j]];
                if (d.n_points)
                    GG_CUDA(cudaMemcpyAsync(draw + (size_t)d.slot * h->pcap, jobs[j].src, d.n_points * sizeof(gg_point), cudaMemcpyHostToDevice,
                                            h->copy_in[KP + (raw_issued & 1)]));
                GG_CUDA(cudaEventRecord(h->raw_ev[raw_issued % h->raw_depth], h->copy_in[KP + (raw_issued & 1)]));
                ++raw_issued;
                ++h->last_raw;
                h->last_raw_bytes += d.n_points * sizeof(gg_point);
                last_raw_bytes = d.n_points * sizeof(gg_point);
                back = j;
                if ((rc = delivered(j))) return rc;
                continue;
            }
            // nothing to enqueue: with the raw queue full (or no mixing) this thread packs a chunk as well
            const auto i0 = std::chrono::steady_clock::now();
            if ((h->host_pack_mix && (bus_free || !h->main_help)) || !h->packer->help()) std::this_thread::yield();
            idle_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - i0).count();
        }
        h->last_pack_us = h->packer->pack_ns.load() / 1000;
        h->last_slot_wait_us = h->packer->slot_wait_ns.load() / 1000;
        h->last_idle_us = idle_ns / 1000;
        pack_guard.armed = false;  // every job is packed or was sent raw
        for (int g = 0; g < h->n_streams; ++g)
            if ((rc = flush(g))) return rc;
        h->batch_parity ^= 1;
    } else {
        // H2D of every 32-byte cloud on its slot's stream, then the kernels of each stream group: everything is
        // stream-ordered, one buffer set is enough
        for (int i = 0; i < count; ++i) {
            const gg_scan_desc& d = scans[i];
            if (d.n_points)
                GG_CUDA(cudaMemcpyAsync(h->view.points + (size_t)d.slot * h->pcap, points[i], d.n_points * sizeof(gg_point), cudaMemcpyHostToDevice,
                                        stream_of(h, d.slot)));
        }
        h->last_raw = (size_t)count;
        for (int i = 0; i < count; ++i) h->last_raw_bytes += scans[i].n_points * sizeof(gg_point);
        if ((rc = run_scans_grouped(h, count, scans, 0))) return rc;
        if (labels_out)
            for (int i = 0; i < count; ++i)
                if (labels_out[i] && scans[i].n_points)
                    GG_CUDA(cudaMemcpyAsync(labels_out[i], h->view.labels + (size_t)scans[i].slot * h->pcap, scans[i].n_points, cudaMemcpyDeviceToHost,
                                            stream_of(h, scans[i].slot)));
    }
    // batch_done: everything enqueued so far on the compute streams and on the label stream
    for (int g = 0; g < h->n_streams; ++g) {
        GG_CUDA(cudaEventRecord(h->batch_ev[g], h->streams[g]));
        GG_CUDA(cudaStreamWaitEvent(h->copy_out, h->batch_ev[g], 0));
    }
    GG_CUDA(cudaEventRecord(h->batch_done[par], h->copy_out));
    h->batch_outstanding[par] = true;
    if (ticket) *ticket = par;
    h->last_feed_us = us_since();
    return GG_OK;
}

int gg_filter_cloud_batch_wait(gg_handle h, int ticket) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (ticket < 0 || ticket > 1) return fail(GG_E_ARG, "bad ticket %d", ticket);
    GG_CUDA(cudaSetDevice(h->device));
    return batch_wait(h, ticket);
}

int gg_filter_cloud_batch(gg_handle h, int count, const gg_scan_desc* scans, const gg_point* const* points, uint8_t* const* labels_out) {
    const auto t_begin = std::chrono::steady_clock::now();
    int rc = gg_filter_cloud_batch_begin(h, count, scans, points, labels_out, nullptr);
    if (rc) return rc;
    rc = gg_synchronize(h);
    h->last_total_us = (size_t)std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t_begin).count();
    return rc;
}

// Timing helpers: make every stream wait for the primary one / the primary one for all others,
// so that a CUDA-event pair on gg_stream() brackets work spread over the handle's streams.
int gg_fork_streams(gg_handle h) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (h->n_streams <= 1) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    cudaEvent_t ev;
    GG_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    GG_CUDA(cudaEventRecord(ev, h->streams[0]));
    for (int g = 1; g < h->n_streams; ++g) GG_CUDA(cudaStreamWaitEvent(h->streams[g], ev, 0));
    GG_CUDA(cudaEventDestroy(ev));
    return GG_OK;
}

int gg_join_streams(gg_handle h) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (h->n_streams <= 1) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    for (int g = 1; g < h->n_streams; ++g) {
        cudaEvent_t ev;
        GG_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        GG_CUDA(cudaEventRecord(ev, h->streams[g]));
        GG_CUDA(cudaStreamWaitEvent(h->streams[0], ev, 0));
        GG_CUDA(cudaEventDestroy(ev));
    }
    return GG_OK;
}

int gg_num_streams(gg_handle h) { return h ? h->n_streams : GG_E_ARG; }

// host-only: the repacking of gg_filter_cloud_batch for one cloud (dst: 14 * ((n + 7) & ~7) bytes,
// 32-byte aligned), chunked like the worker threads do it -- exported for the CPU tests
static int pack_whole_cloud(const gg_point* src, size_t n, unsigned char* dst, bool cached) {
    if ((!src && n) || !dst) return GG_E_ARG;
    size_t i0 = 0;
    do {
        const size_t i1 = std::min(n, i0 + HostPacker::kChunk);
        HostPacker::pack_range(src, n, dst, i0, i1, cached);
        i0 = i1;
    } while (i0 < n);
    return GG_OK;
}
int gg_host_pack_cloud(const gg_point* src, size_t n, unsigned char* dst) { return pack_whole_cloud(src, n, dst, false); }
// same with plain (cache-allocating) stores
int gg_host_pack_cloud_cached(const gg_point* src, size_t n, unsigned char* dst) { return pack_whole_cloud(src, n, dst, true); }

// host-only self-test of the packer pool (no CUDA): `rounds` batches of n_jobs clouds go through a ring of
// `ring_slots` staging slots; this thread plays the feeder of gg_filter_cloud_batch_begin -- it checks every packed
// cloud against the single-threaded packing, "completes" its copy `lag` jobs later (so packers have to wait for
// slots), takes some jobs away from the back like the raw path does, and cancels the last batch half way.
// Returns 0, or a negative code telling which check failed.
int gg_host_packer_selftest(int threads, int n_jobs, size_t n_points, int ring_slots, int rounds, int lag) {
    if (threads < 1 || n_jobs < 1 || ring_slots < 2 || rounds < 1 || lag < 0 || lag >= ring_slots) return GG_E_ARG;
    const size_t n_pad = (n_points + 7) & ~(size_t)7, stride = 14 * n_pad + 64;
    std::vector<std::vector<gg_point>> src(n_jobs);
    std::vector<std::vector<unsigned char>> want(n_jobs);
    uint32_t lcg = 12345u;
    for (int j = 0; j < n_jobs; ++j) {
        const size_t n = n_points - (size_t)(j % 5);  // ragged sizes
        src[j].resize(n);
        unsigned char* raw = reinterpret_cast<unsigned char*>(src[j].data());
        for (size_t b = 0; b < n * sizeof(gg_point); ++b) {
            lcg = lcg * 1664525u + 1013904223u;
            raw[b] = (unsigned char)(lcg >> 24);
        }
        want[j].assign(stride + 32, 0);
        unsigned char* w = want[j].data() + ((32 - (reinterpret_cast<uintptr_t>(want[j].data()) & 31)) & 31);
        pack_whole_cloud(src[j].data(), n, w, false);
    }
    auto want_ptr = [&](int j) { return want[j].data() + ((32 - (reinterpret_cast<uintptr_t>(want[j].data()) & 31)) & 31); };
    std::vector<unsigned char> ring_mem((size_t)ring_slots * stride + 64);
    unsigned char* ring = ring_mem.data() + ((64 - (reinterpret_cast<uintptr_t>(ring_mem.data()) & 63)) & 63);
    HostPacker packer(threads);
    packer.set_ring(ring, stride, ring_slots);
    uint64_t issued = 0;
    for (int round = 0; round < rounds; ++round) {
        std::vector<PackJob> jobs(n_jobs);
        for (int j = 0; j < n_jobs; ++j) {
            jobs[j].src = src[j].data();
            jobs[j].n = src[j].size();
        }
        const bool cancel_round = round == rounds - 1;
        const uint64_t base = issued;
        packer.start(&jobs, base);
        int front = 0, back = n_jobs, spins = 0;
        while (front < back) {
            if (issued >= (uint64_t)lag) packer.copied.store(issued - (uint64_t)lag, std::memory_order_release);
            if (cancel_round && front >= n_jobs / 2) {
                packer.cancel();
                break;
            }
            if (packer.packed(jobs[front])) {
                const size_t np = (jobs[front].n + 7) & ~(size_t)7;
                if (std::memcmp(packer.slot_of(base + front), want_ptr(front), 14 * np) != 0) return -100 - front;
                ++issued;
                ++front;
                spins = 0;
                continue;
            }
            if ((front + round) % 3 == 0) {
                const int j = packer.claim_raw_from_back();
                if (j >= 0) {
                    if (j != back - 1) return -50;
                    back = j;
                    continue;
                }
            }
            if (!packer.help()) std::this_thread::yield();
            if (++spins > 200000000) return -60;  // stuck
        }
        packer.copied.store(issued, std::memory_order_release);  // all copies of this batch "done"
    }
    return GG_OK;
}


// number of host threads that repack clouds in gg_filter_cloud_batch (0: packing disabled or not used yet)
int gg_host_pack_threads(gg_handle h) { return (h && h->host_pack && h->packer) ? h->packer->threads() + 1 : 0; }

int gg_last_batch_transfer(gg_handle h, size_t info[9]) {
    if (!h || !info) return fail(GG_E_ARG, "null argument");
    info[0] = h->last_packed;
    info[1] = h->last_raw;
    info[2] = h->last_packed_bytes;
    info[3] = h->last_raw_bytes;
    info[4] = h->last_feed_us;
    info[5] = h->last_total_us;
    info[6] = h->last_pack_us;
    info[7] = h->last_slot_wait_us;
    info[8] = h->last_idle_us;
    return GG_OK;
}

int gg_get_layer(gg_handle h, int slot, const char* name, float* dst) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!dst) return fail(GG_E_ARG, "null dst");
    GG_CUDA(cudaSetDevice(h->device));
    const size_t bytes = (size_t)h->view.k.N2 * sizeof(float);
    if (name && std::strcmp(name, "expectedPoints") == 0) {
        GG_CUDA(cudaMemcpy(dst, h->view.expected, bytes, cudaMemcpyDeviceToHost));
        return GG_OK;
    }
    int idx;
    if ((rc = layer_index(h, slot, name, &idx))) return rc;
    if ((rc = gg_synchronize(h))) return rc;
    GG_CUDA(cudaMemcpy(dst, h->view.layer(slot, idx), bytes, cudaMemcpyDeviceToHost));
    return GG_OK;
}

int gg_set_layer(gg_handle h, int slot, const char* name, const float* src) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!src) return fail(GG_E_ARG, "null src");
    GG_CUDA(cudaSetDevice(h->device));
    int idx;
    if ((rc = layer_index(h, slot, name, &idx))) return rc;
    if ((rc = gg_synchronize(h))) return rc;
    GG_CUDA(cudaMemcpy(h->view.layer(slot, idx), src, (size_t)h->view.k.N2 * sizeof(float), cudaMemcpyHostToDevice));
    return GG_OK;
}

int gg_layer_device_ptr(gg_handle h, int slot, const char* name, void** dptr) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!dptr) return fail(GG_E_ARG, "null dptr");
    int idx;
    if ((rc = layer_index(h, slot, name, &idx))) return rc;
    *dptr = h->view.layer(slot, idx);
    return GG_OK;
}

namespace {
// gg_get_layers_to_device (import = false) / gg_set_layers_from_device (import = true): one k_layer_copy per stream
// group with slots in the batch.
int layer_transfer(gg_handle h, int count, const int* slots, int n_names, const char* const* names, float* buf, bool import, void* stream) {
    gg::LayerList list{};
    int points_at = -1, rc;
    const size_t bytes = h ? (size_t)count * n_names * h->view.k.N2 * sizeof(float) : 0;
    if ((rc = check_slot_batch(h, count, slots, n_names, names, {{buf, bytes, alignof(float), true, "buffer"}}, &list, &points_at)) ||
        count == 0 || n_names == 0)
        return rc;
    // an import must not write one layer of a slot twice ("points" is also "obstacles" or "count")
    if (import && points_at >= 0)
        for (int i = 0; i < count; ++i) {
            const int p = points_layer(h, slots[i]);
            for (int l = 0; l < n_names; ++l)
                if (list.idx[l] == p)
                    return fail(GG_E_ARG, "slot %d: '%s' and 'points' are the same layer", slots[i], names[l]);
        }
    return enqueue_slot_batch(h, count, slots, stream, [&](const Staging& e, cudaStream_t st) {
        return gg::launch_layer_copy(h->view, e.dp, e.m, list, buf, import, st, h->prof);
    });
}
}  // namespace

int gg_get_layers_to_device(gg_handle h, int count, const int* slots, int n_names, const char* const* names, float* dst, void* stream) {
    return layer_transfer(h, count, slots, n_names, names, dst, false, stream);
}

int gg_set_layers_from_device(gg_handle h, int count, const int* slots, int n_names, const char* const* names, const float* src,
                              void* stream) {
    return layer_transfer(h, count, slots, n_names, names, const_cast<float*>(src), true, stream);
}

// Terrain lookups: one k_sample_layers per stream group with non-empty sets in the batch.
int gg_sample_layers_to_device(gg_handle h, int count, const int* slots, const gg_positions* queries, int n_names, const char* const* names,
                               int mode, void* stream) {
    gg::LayerList list{};
    int points_at = -1, rc;
    if ((rc = check_slot_batch(h, count, slots, n_names, names, {}, &list, &points_at)) || count == 0 || n_names == 0) return rc;
    if (!queries) return fail(GG_E_ARG, "null queries");
    if (mode != GG_SAMPLE_NEAREST && mode != GG_SAMPLE_LINEAR) return fail(GG_E_ARG, "unknown sample mode %d", mode);
    const gg::View& v = h->view;
    const void* arena = v.layers;
    const size_t arena_bytes = (size_t)h->n_slots * v.n_layers * v.k.N2 * sizeof(float);
    std::vector<ByteRange>& ranges = h->range_scratch;
    ranges.clear();
    size_t total = 0;
    for (int k = 0; k < count; ++k) {
        const gg_positions& q = queries[k];
        if (q.n == 0) continue;
        if (q.n > (size_t)INT32_MAX) return fail(GG_E_ARG, "set %d: %zu positions, at most %d", k, q.n, INT32_MAX);
        if (!q.data || !q.dst) return fail(GG_E_ARG, "set %d: null data or dst", k);
        if (q.point_step < 8 || q.point_step % 4) return fail(GG_E_ARG, "set %d: point_step %d is not a multiple of 4 of at least 8", k, q.point_step);
        if (q.off_x < 0 || q.off_y < 0 || q.off_x % 4 || q.off_y % 4 || q.off_x > q.point_step - 4 || q.off_y > q.point_step - 4)
            return fail(GG_E_ARG, "set %d: offsets (%d, %d) are not multiples of 4 inside point_step %d", k, q.off_x, q.off_y, q.point_step);
        if (reinterpret_cast<uintptr_t>(q.data) % 4 || reinterpret_cast<uintptr_t>(q.dst) % 4 || reinterpret_cast<uintptr_t>(q.cell) % 4)
            return fail(GG_E_ARG, "set %d: data, dst or cell is not 4-byte aligned", k);
        const size_t dst_bytes = (size_t)n_names * q.n * sizeof(float), cell_bytes = q.n * sizeof(int32_t);
        if (ranges_overlap(q.dst, dst_bytes, arena, arena_bytes) || ranges_overlap(q.cell, cell_bytes, arena, arena_bytes))
            return fail(GG_E_ARG, "set %d: an output overlaps the handle's layers", k);
        const uintptr_t data = reinterpret_cast<uintptr_t>(q.data), dst = reinterpret_cast<uintptr_t>(q.dst);
        ranges.push_back({data, data + q.n * (size_t)q.point_step, k, false});
        ranges.push_back({dst, dst + dst_bytes, k, true});
        if (q.cell) ranges.push_back({reinterpret_cast<uintptr_t>(q.cell), reinterpret_cast<uintptr_t>(q.cell) + cell_bytes, k, true});
        total += q.n;
    }
    // Outputs must not overlap any range; inputs may share memory.  Sorted by start, a range overlaps an earlier one iff
    // it starts below the largest end among them, so one sweep keeps the farthest-reaching range and the farthest output.
    std::sort(ranges.begin(), ranges.end(), [](const ByteRange& a, const ByteRange& b) { return a.begin < b.begin; });
    const ByteRange *far_any = nullptr, *far_out = nullptr;
    for (const ByteRange& r : ranges) {
        const ByteRange* o = r.output ? far_any : far_out;
        if (o && o->end > r.begin)
            return fail(GG_E_ARG, "set %d: %s overlaps %s of set %d", r.set, r.output ? "an output" : "the positions",
                        o->output ? "an output" : "the positions", o->set);
        if (!far_any || r.end > far_any->end) far_any = &r;
        if (r.output && (!far_out || r.end > far_out->end)) far_out = &r;
    }
    if (total == 0) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    auto fill = [&](int i, Staging& e) {
        const gg_positions& q = queries[i];
        const SlotState& s = h->slots[slots[i]];
        gg::SlotParams& p = e.hp[e.m];
        std::memset(&p, 0, sizeof(p));
        p.slot = slots[i];
        p.pos = i;
        p.points_layer = points_layer(h, slots[i]);
        p.px = s.px;
        p.py = s.py;
        e.position = true;
        p.n_points = (int)q.n;
        gg::QueryDesc& d = e.hquery[e.m];
        std::memset(&d, 0, sizeof(d));
        d.data = static_cast<const unsigned char*>(q.data);
        d.dst = q.dst;
        d.cell = q.cell;
        d.point_step = q.point_step;
        d.off_x = q.off_x;
        d.off_y = q.off_y;
        e.query = true;
        return q.n > 0;
    };
    auto launch = [&](const Staging& e, cudaStream_t st) {
        return gg::launch_sample(h->view, e.dp, e.dquery, e.m, e.max_points, list, mode, st, h->prof);
    };
    return run_groups(h, count, slots, true, static_cast<cudaStream_t>(stream), fill, launch);
}

// Point classes and heights: one k_point_info per stream group with something to write.
int gg_point_info_to_device(gg_handle h, int count, const int* slots, const gg_point_info* outs, void* stream) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (count < 0) return fail(GG_E_ARG, "negative count");
    if (count == 0) return GG_OK;
    if (!slots || !outs) return fail(GG_E_ARG, "null argument");
    int rc;
    if ((rc = check_slots(h, count, slots))) return rc;
    const gg::View& v = h->view;
    const void* arena = v.layers;
    const size_t arena_bytes = (size_t)h->n_slots * v.n_layers * v.k.N2 * sizeof(float);
    std::vector<ByteRange>& ranges = h->range_scratch;
    ranges.clear();
    for (int k = 0; k < count; ++k) {
        const int slot = slots[k];
        const SlotState& s = h->slots[slot];
        if ((rc = check_completed_scan(h, slot))) return rc;
        if (s.moved_since_scan) return fail(GG_E_STATE, "slot %d: the map moved since its last scan (the cell indices are stale)", slot);
        if (s.device_rolled)
            return fail(GG_E_STATE, "slot %d: a device roll since its last scan may have moved the map (the cell indices may be stale)", slot);
        const gg_point_info& o = outs[k];
        if (reinterpret_cast<uintptr_t>(o.codes) % 4 || reinterpret_cast<uintptr_t>(o.height) % 4)
            return fail(GG_E_ARG, "slot %d: codes or height is not 4-byte aligned", slot);
        const size_t bytes = s.scan_points * sizeof(uint32_t);
        for (const void* p : {static_cast<const void*>(o.codes), static_cast<const void*>(o.height)}) {
            if (!p || !bytes) continue;
            if (ranges_overlap(p, bytes, arena, arena_bytes)) return fail(GG_E_ARG, "slot %d: an output overlaps the handle's layers", slot);
            ranges.push_back({reinterpret_cast<uintptr_t>(p), reinterpret_cast<uintptr_t>(p) + bytes, k, true});
        }
    }
    // every range is an output: sorted by start, a range overlaps an earlier one iff it starts below their largest end
    std::sort(ranges.begin(), ranges.end(), [](const ByteRange& a, const ByteRange& b) { return a.begin < b.begin; });
    const ByteRange* far = nullptr;
    for (const ByteRange& r : ranges) {
        if (far && far->end > r.begin) return fail(GG_E_ARG, "an output of slot %d overlaps an output of slot %d", slots[r.set], slots[far->set]);
        if (!far || r.end > far->end) far = &r;
    }
    if (ranges.empty()) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    // the staging of the destinations, parallel to the ring, on first use (a handle that never asks has none)
    if (!h->d_pinfo && (rc = dev_alloc(h, &h->d_pinfo, (size_t)kRing * h->n_slots))) return rc;
    if (!h->h_pinfo)
        GG_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h->h_pinfo), sizeof(gg::PointInfoDest) * kRing * h->n_slots, cudaHostAllocDefault));
    auto fill = [&](int i, Staging& e) {
        const SlotState& s = h->slots[slots[i]];
        const gg_point_info& o = outs[i];
        const bool write = s.scan_points > 0 && (o.codes || o.height);
        gg::SlotParams& p = e.hp[e.m];
        std::memset(&p, 0, sizeof(p));
        p.slot = slots[i];
        p.pos = i;
        p.n_points = write ? (int)s.scan_points : 0;
        gg::PointInfoDest& d = e.hpinfo[e.m];
        d.codes = o.codes;
        d.height = o.height;
        e.pinfo = true;
        return write;
    };
    auto launch = [&](const Staging& e, cudaStream_t st) { return gg::launch_point_info(h->view, e.dp, e.dpinfo, e.m, e.max_points, st, h->prof); };
    return run_groups(h, count, slots, true, static_cast<cudaStream_t>(stream), fill, launch);
}

// Poses from device memory: per stream group one k_pose_resolve over the group's slots, then (with xy) the roll kernels
// on the same staging entry.
int gg_update_poses_from_device(gg_handle h, int count, const int* slots, const gg_device_poses* poses, int32_t* dev_moved, void* stream) {
    if (!h) return fail(GG_E_ARG, "null handle");
    if (count < 0) return fail(GG_E_ARG, "negative count");
    if (count == 0) return GG_OK;
    if (!slots || !poses) return fail(GG_E_ARG, "null argument");
    int rc;
    if ((rc = check_slots(h, count, slots))) return rc;
    const gg_device_poses& in = *poses;
    if (!in.xy != !in.T_base_from_map) return fail(GG_E_ARG, "xy and T_base_from_map must both be given or both be NULL");
    if (!in.origin != !in.base_z) return fail(GG_E_ARG, "origin and base_z must both be given or both be NULL");
    auto misaligned = [](const void* p, size_t a) { return reinterpret_cast<uintptr_t>(p) % a != 0; };
    if (misaligned(in.xy, 8) || misaligned(in.T_base_from_map, 8) || misaligned(in.base_z, 8))
        return fail(GG_E_ARG, "xy, T_base_from_map or base_z is not 8-byte aligned");
    if (misaligned(in.origin, 4) || misaligned(dev_moved, 4)) return fail(GG_E_ARG, "origin or dev_moved is not 4-byte aligned");
    const size_t n = (size_t)count, moved_bytes = n * sizeof(int32_t);
    const gg::View& v = h->view;
    if (ranges_overlap(dev_moved, moved_bytes, v.layers, (size_t)h->n_slots * v.n_layers * v.k.N2 * sizeof(float)))
        return fail(GG_E_ARG, "dev_moved overlaps the handle's layers");
    if (ranges_overlap(dev_moved, moved_bytes, in.xy, n * 2 * sizeof(double)) || ranges_overlap(dev_moved, moved_bytes, in.T_base_from_map, n * 12 * sizeof(double)) ||
        ranges_overlap(dev_moved, moved_bytes, in.origin, n * 3 * sizeof(float)) || ranges_overlap(dev_moved, moved_bytes, in.base_z, n * sizeof(double)))
        return fail(GG_E_ARG, "dev_moved overlaps the poses");
    if (!in.xy && !in.origin) return GG_OK;
    GG_CUDA(cudaSetDevice(h->device));
    // the device tables and the staging of the pose bits, on first use (a handle that never asks has none)
    const size_t S = (size_t)h->n_slots;
    if (!h->poses.position && (rc = dev_alloc(h, &h->poses.position, S))) return rc;
    if (!h->poses.scan_pose && (rc = dev_alloc(h, &h->poses.scan_pose, S))) return rc;
    if (!h->d_pose_bits && (rc = dev_alloc(h, &h->d_pose_bits, (size_t)kRing * S))) return rc;
    if (!h->h_pose_bits) GG_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h->h_pose_bits), sizeof(int) * kRing * S, cudaHostAllocDefault));
    const gg::DevicePoses dp{in.xy, in.T_base_from_map, in.origin, in.base_z, dev_moved};
    auto fill = [&](int i, Staging& e) {
        SlotState& s = h->slots[slots[i]];
        gg::SlotParams& p = e.hp[e.m];
        std::memset(&p, 0, sizeof(p));
        p.slot = slots[i];
        p.pos = i;
        p.px = s.px;   // the position k_pose_resolve starts from, unless the device table holds it
        p.py = s.py;
        e.hbits[e.m] = s.device_position ? gg::POSE_POSITION : 0;
        e.pose_bits = true;
        if (in.xy) s.device_position = s.device_rolled = true;
        if (in.origin) s.device_scan_pose = true;
        return true;
    };
    auto launch = [&](const Staging& e, cudaStream_t st) {
        int launched = gg::launch_pose_resolve(h->view, h->poses, e.dp, e.dbits, e.m, dp, st, h->prof);
        if (in.xy) launched += gg::launch_roll(h->view, e.dp, e.m, st, h->prof);
        return launched;
    };
    return run_groups(h, count, slots, true, static_cast<cudaStream_t>(stream), fill, launch);
}

int gg_last_scan_points(gg_handle h, int slot, size_t* n_points) {
    int rc = check_slot(h, slot);
    if (rc) return rc;
    if (!n_points) return fail(GG_E_ARG, "null argument");
    *n_points = h->slots[slot].scan_points;
    return GG_OK;
}

}  // extern "C"
