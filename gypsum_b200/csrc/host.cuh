// What the two halves of the C ABI's host layer share: engine.cu (the engine, its IQ and acquisition) and receiver.cu
// (the trackers and their receiver chain).  Host code only.
#pragma once
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/gypsum_b200.h"
#include "kernels.cuh"

namespace gb::capi {

struct DeviceMemory {
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
    static void free(void* p) { cudaFree(p); }
};
struct PinnedMemory {
    static cudaError_t alloc(void** p, size_t bytes) { return cudaMallocHost(p, bytes); }
    static void free(void* p) { cudaFreeHost(p); }
};

// A growable array of device (DeviceMemory) or page-locked host (PinnedMemory) memory that frees itself.  ensure() keeps
// the contents only while the array does not have to grow.
template <class T, class Memory>
struct Buf {
    T* p = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    Buf(Buf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    ~Buf() { release(); }
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        release();
        size_t want = std::max(n, static_cast<size_t>(16));
        cudaError_t e = Memory::alloc(reinterpret_cast<void**>(&p), want * sizeof(T));
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) Memory::free(p);
        p = nullptr;
        cap = 0;
    }
};
template <class T>
using DevBuf = Buf<T, DeviceMemory>;
template <class T>
using PinnedBuf = Buf<T, PinnedMemory>;

}  // namespace gb::capi

struct gb200_engine {
    int device = 0, fs = 0, N = 0, s = 0, num_sms = 132;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    gb::capi::DevBuf<float2> tw1, tw2, crep, crep1023, iq_own, spec, d_replica;
    gb::capi::DevBuf<uint8_t> chips;
    gb::capi::DevBuf<double> d_doppler;
    gb::capi::DevBuf<int> d_ints;
    gb::capi::DevBuf<gb::CellRecord> d_records;
    gb::capi::DevBuf<float> d_profile;
    struct {  // gb200_detect, the on-device satellite search
        gb::capi::DevBuf<gb::RefineState> state;
        gb::capi::DevBuf<double> d_doppler;
        gb::capi::DevBuf<gb::CellRecord> d_records;
        gb::capi::DevBuf<int> d_ints, d_cell_prn;
        gb::capi::DevBuf<gb::RefineResult> d_results;
        gb::capi::PinnedBuf<int> h_ints, h_cell_prn;
        gb::capi::PinnedBuf<gb::RefineResult> h_results;
    } search;
    gb::capi::PinnedBuf<float2> h_iq, h_replica;
    gb::capi::PinnedBuf<gb::CellRecord> h_records;
    gb::capi::PinnedBuf<int> h_ints;
    gb::capi::PinnedBuf<double> h_doubles;
    gb::capi::PinnedBuf<float> h_profile;
    struct {  // the grid axes d_doppler[0..] and d_ints[0..] hold, until a list-mode call reuses those buffers
        std::vector<double> dop;
        std::vector<int> prn;
        bool valid = false;
    } grid_axes;
    int n_prn = 0;
    const float2* iq = nullptr;
    int64_t iq_samples = 0;
    int64_t launches = 0;
    // read from the environment at gb200_create: GB200_SPEC_BUDGET_MB, GB200_L2_WINDOW_MB, GB200_L2_WINDOW_MIN_GROUPS
    size_t spec_budget_bytes = 512u << 20, l2_window_bytes = 16u << 20;
    int l2_window_min_groups = 2;
    bool timing = false;
    int fused = -1;  // acquire_cells kernel choice: -1 automatic, 0 doppler_spectra + correlate_cells, 1 fused block-per-cell
    bool fused_configured = false;
    gb::capi::DevBuf<gb::BestRecord> d_best;
    gb::capi::PinnedBuf<gb::BestRecord> h_best;
    // gb200_acquire_grid_host: one CUDA graph (copy-in, doppler_spectra, correlate_cells, copy-out) per grid shape
    struct HostGraph {
        // Everything a captured graph bakes in: the grid's shape and axes, and every buffer it reads or writes.
        struct Key {
            int n_blocks = 0, M = 0, P = 0, D = 0, kind = 0;
            std::vector<double> dop;
            std::vector<int> prn;
            const void *iq_dev = nullptr, *rec_dev = nullptr, *iq_stage = nullptr, *rec_stage = nullptr, *spec = nullptr;
            const void *d_dop = nullptr, *d_prn = nullptr, *crep = nullptr, *crep1023 = nullptr;  // what the captured kernels dereference besides the above
            const void* rec_target = nullptr;  // where the captured correlate kernel stores its records
            cudaStream_t stream = nullptr;
            auto ids() const {
                return std::tie(n_blocks, M, P, D, kind, iq_dev, rec_dev, iq_stage, rec_stage, spec, d_dop, d_prn, crep, crep1023, rec_target,
                                stream);
            }
            // the axes compare bit for bit, as the device copies of them do (upload_grid_axes)
            bool operator==(const Key& o) const {
                return ids() == o.ids() && dop.size() == o.dop.size() && prn == o.prn &&
                       memcmp(dop.data(), o.dop.data(), sizeof(double) * dop.size()) == 0;
            }
        } key;
        cudaGraphExec_t exec = nullptr;
        int seen = 0;
    } hg;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev[2];
    size_t ev_used[2] = {0, 0};
    std::string err;

    ~gb200_engine() {  // the buffers free themselves
        if (hg.exec) cudaGraphExecDestroy(hg.exec);
        for (auto& pool : ev)
            for (auto& pr : pool) {
                cudaEventDestroy(pr.first);
                cudaEventDestroy(pr.second);
            }
        if (own_stream) cudaStreamDestroy(own_stream);
    }
};

#define GB_FAIL(e, code, ...)                        \
    do {                                             \
        char buf_[512];                              \
        snprintf(buf_, sizeof(buf_), __VA_ARGS__);   \
        (e)->err = buf_;                             \
        return code;                                 \
    } while (0)

#define GB_CUDA(e, expr)                                                                                   \
    do {                                                                                                   \
        cudaError_t ce_ = (expr);                                                                          \
        if (ce_ != cudaSuccess) {                                                                          \
            cudaGetLastError();                                                                            \
            GB_FAIL(e, GB200_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(ce_), __FILE__, __LINE__); \
        }                                                                                                  \
    } while (0)

#define GB_TRY(expr)                       \
    do {                                   \
        const int rc_ = (expr);            \
        if (rc_ != GB200_OK) return rc_;   \
    } while (0)

// One kernel launch: the optional timing bracket of kernel class `which` (0 doppler_spectra, 1 correlate, -1 untimed),
// the error check and the launch count (gb200_launch_count).
#define GB_LAUNCH(e, which, expr)                    \
    do {                                             \
        {                                            \
            gb::capi::TimedLaunch tl_((e), (which)); \
            GB_CUDA((e), expr);                      \
        }                                            \
        (e)->launches++;                             \
    } while (0)

namespace gb::capi {

// optional event bracket around one kernel launch (measurement aid, off by default)
struct TimedLaunch {
    gb200_engine* e;
    int which;
    cudaEvent_t stop = nullptr;
    TimedLaunch(gb200_engine* e_, int which_) : e(e_), which(which_) {
        if (!e->timing || which < 0) return;
        auto& pool = e->ev[which];
        if (e->ev_used[which] == pool.size()) {
            cudaEvent_t a, b;
            if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return;
            pool.emplace_back(a, b);
        }
        auto& pr = pool[e->ev_used[which]++];
        cudaEventRecord(pr.first, e->stream);
        stop = pr.second;
    }
    ~TimedLaunch() {
        if (stop) cudaEventRecord(stop, e->stream);
    }
};

// Argument rules shared by the entry points, one function each.
inline int check_replicas(gb200_engine* e) {
    if (e->n_prn == 0) GB_FAIL(e, GB200_ESTATE, "no PRN replicas loaded (gb200_set_replicas)");
    return GB200_OK;
}

inline int check_prns(gb200_engine* e, const int32_t* prn_idx, int n) {
    for (int i = 0; i < n; ++i)
        if (prn_idx[i] < 0 || prn_idx[i] >= e->n_prn) GB_FAIL(e, GB200_EINVAL, "prn index %d out of range", prn_idx[i]);
    return GB200_OK;
}

inline int check_iq(gb200_engine* e, int n_ms) {
    if (!e->iq) GB_FAIL(e, GB200_ESTATE, "no IQ loaded (gb200_upload_iq / gb200_bind_iq_device)");
    if (n_ms < 1) GB_FAIL(e, GB200_EINVAL, "need at least one whole millisecond of samples");
    return GB200_OK;
}

inline int check_samples(gb200_engine* e, int n_ms) {
    if (static_cast<int64_t>(n_ms) * e->N > e->iq_samples)
        GB_FAIL(e, GB200_EINVAL, "need %lld samples, %lld loaded", static_cast<long long>(n_ms) * e->N,
                static_cast<long long>(e->iq_samples));
    return GB200_OK;
}

// Whether p is page-locked host memory, which the DMA engine reads and writes directly; *alias (optional) receives its
// device address.
inline bool is_pinned(const void* p, void** alias = nullptr) {
    cudaPointerAttributes attr{};
    const bool pinned = cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (alias) *alias = pinned ? attr.devicePointer : nullptr;
    return pinned;
}

// Copies n host elements into the pinned buffer stage (grown to fit) and points src at the copy.  No copy in flight may
// still read stage: the caller synchronises first, or owns the buffer.
template <class T>
cudaError_t stage_in(PinnedBuf<T>& stage, const T*& src, size_t n) {
    cudaError_t ce = stage.ensure(std::max<size_t>(n, 1));
    if (ce != cudaSuccess) return ce;
    memcpy(stage.p, src, n * sizeof(T));
    src = stage.p;
    return cudaSuccess;
}

// Puts n host elements on the device at dst through the pinned buffer stage (see stage_in).
template <class T>
int upload(gb200_engine* e, T* dst, const T* src, size_t n, PinnedBuf<T>& stage) {
    GB_CUDA(e, stage_in(stage, src, n));
    GB_CUDA(e, cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, e->stream));
    return GB200_OK;
}

// Brings n device elements to dst and waits for them (and for everything enqueued before): straight DMA when dst is
// pinned, else through the pinned buffer stage.
template <class T>
int download(gb200_engine* e, T* dst, const T* src, size_t n, PinnedBuf<T>& stage) {
    T* to = dst;
    if (!is_pinned(dst)) {
        GB_CUDA(e, stage.ensure(n));
        to = stage.p;
    }
    GB_CUDA(e, cudaMemcpyAsync(to, src, n * sizeof(T), cudaMemcpyDeviceToHost, e->stream));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    if (to != dst) memcpy(dst, to, n * sizeof(T));
    return GB200_OK;
}

}  // namespace gb::capi
