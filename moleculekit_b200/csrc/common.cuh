// common.cuh -- handle, scratch and error plumbing shared by the mkb200 translation units.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <mutex>
#include <string>

#include "mkb200.h"

namespace mkb {

enum ScratchSlot {
    S_DESC = 0,     // device copy of per-grid descriptors
    S_ITEM_CELL,    // per (grid, atom) item: cell id / slot
    S_ITEM_SLOT,
    S_CELL_COUNT,   // per cell counters, then exclusive offsets
    S_CELL_START,
    S_SCAN_TMP,     // cub temp storage
    S_SORT_PX, S_SORT_PY, S_SORT_PZ, S_SORT_S2, S_SORT_MASK, S_SORT_SRC,
    S_PT_S2,        // points path: per (atom, channel) sigma^2
    S_PT_BUCKET,    // points path: bucket offsets
    S_PT_ORDER,     // points path: atom order
    S_ROWCNT,       // contacts: per-row counts
    S_COM,          // reductions: centres of mass
    S_TILE_TOTAL,   // occupancy fast paths: halo atom count per tile / per block
    S_BLOCK_BASE,   // occupancy warp kernel: first block id of every grid
    S_K4_BALLOTS,   // contacts: hit masks of the count pass, reused by the fill pass
    S_BAND_BITMAP,  // occupancy run kernel: one bit per voxel whose gate decision is re-done in float64
    S_QUEUE,        // occupancy run kernel: block queue counter
    S_FIX_LIST,     // occupancy run kernel: voxels re-evaluated in float64 (count + list)
    S_BLK_ENT,      // occupancy run kernel: per-block candidate lists
    S_BLK_SLOTS,    // occupancy run kernel: the slot of every (atom, block) insertion
    S_NSLOTS
};

struct Scratch {
    void *ptr = nullptr;
    size_t cap = 0;
};

}  // namespace mkb

struct mkb_ctx {
    int device = 0;
    std::string err;
    mkb::Scratch scratch[mkb::S_NSLOTS];
    int64_t launches = 0;
    const char *last_kernel = "";  // main kernel of the most recent occupancy / distance call (bench.py's roofline.kernel)
    int sm_count = 132;
    // optional per-kernel timing (bench.py roofline): events recorded on the launch stream
    bool timing = false;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};  // before prep, before main kernel, after main kernel
    // One handle = one set of grow-only scratch buffers.  Entry points may be called from several host threads and on
    // several streams: the mutex serialises the host side of a call, and a call on a stream other than the previous one's
    // first waits for the event recorded at the end of the previous call, so two calls never share scratch in flight.
    std::recursive_mutex mtx;
    cudaEvent_t order_ev = nullptr;
    cudaStream_t order_stream = nullptr;
    bool order_valid = false;
    // page-locked staging for the small per-call host -> device uploads (grid descriptors): a pageable cudaMemcpyAsync
    // stages through the driver and costs tens of microseconds of host time per call
    static constexpr int N_STAGE = 4;  // a ring, so the host can run several calls ahead of the device
    void *host_stage[N_STAGE] = {};
    size_t host_stage_cap[N_STAGE] = {};
    cudaEvent_t stage_ev[N_STAGE] = {};
    int stage_next = 0;
    // side stream of the occupancy run path (gate-band pre-pass beside the list build)
    cudaStream_t aux_stream = nullptr, aux_stream2 = nullptr;
    bool index_pending = false;  // mkb_occupancy_grid_batch_to_host: the block index is on its way to the host (aux_ev[3])
    cudaEvent_t aux_ev[2 + 16] = {};  // band fork / join, one per chunk of the list-build pipeline
    // K4: the count call leaves one ballot word per (row, 32 columns); the fill call that follows with the SAME arguments
    // reads them instead of evaluating every distance a second time
    struct K4Key {
        const void *coords = nullptr, *box = nullptr, *sel1 = nullptr, *sel2 = nullptr, *chains = nullptr;
        long long F = 0, n1 = 0, n2 = 0, fs = 0, fsb = 0;
        int selfdist = 0, pbc = 0;
        unsigned thr_bits = 0;
        bool valid = false;
        bool same(const K4Key &o) const {
            return valid && o.valid && coords == o.coords && box == o.box && sel1 == o.sel1 && sel2 == o.sel2 &&
                   chains == o.chains && F == o.F && n1 == o.n1 && n2 == o.n2 && fs == o.fs && fsb == o.fsb &&
                   selfdist == o.selfdist && pbc == o.pbc && thr_bits == o.thr_bits;
        }
    } k4_key;
};

namespace mkb {

inline int fail(mkb_ctx *h, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf;
    return code;
}

#define MKB_CUDA(h, expr)                                                                            \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess)                                                                       \
            return mkb::fail((h), MKB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                             __FILE__, __LINE__);                                                    \
    } while (0)

// Grow-only scratch.  cudaFree synchronises the device, so a buffer still in use by in-flight work is never
// pulled from under it.
inline int scratch_get(mkb_ctx *h, ScratchSlot s, size_t bytes, void **out) {
    Scratch &sc = h->scratch[s];
    if (bytes > sc.cap) {
        if (sc.ptr) MKB_CUDA(h, cudaFree(sc.ptr));
        sc.ptr = nullptr;
        sc.cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&sc.ptr, want);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            return fail(h, MKB_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
        }
        sc.cap = want;
    }
    *out = sc.ptr;
    return MKB_OK;
}

// page-locked staging buffer of `bytes` (next slot of the ring); waits until the upload that last used the slot has left the
// host.  The caller records *ev on its stream after enqueuing the copy.
inline int host_stage_get(mkb_ctx *h, size_t bytes, void **out, cudaEvent_t **ev) {
    const int k = h->stage_next;
    h->stage_next = (k + 1) % mkb_ctx::N_STAGE;
    if (h->stage_ev[k]) MKB_CUDA(h, cudaEventSynchronize(h->stage_ev[k]));
    else MKB_CUDA(h, cudaEventCreateWithFlags(&h->stage_ev[k], cudaEventDisableTiming));
    if (bytes > h->host_stage_cap[k]) {
        if (h->host_stage[k]) MKB_CUDA(h, cudaFreeHost(h->host_stage[k]));
        h->host_stage[k] = nullptr;
        h->host_stage_cap[k] = 0;
        const size_t want = bytes + bytes / 2 + 4096;
        MKB_CUDA(h, cudaHostAlloc(&h->host_stage[k], want, cudaHostAllocDefault));
        h->host_stage_cap[k] = want;
    }
    *out = h->host_stage[k];
    *ev = &h->stage_ev[k];
    return MKB_OK;
}

template <typename T>
inline int scratch_get(mkb_ctx *h, ScratchSlot s, size_t count, T **out) {
    void *p = nullptr;
    int rc = scratch_get(h, s, count * sizeof(T), &p);
    *out = static_cast<T *>(p);
    return rc;
}

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() {
        int cur = -1;
        if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
    }
};

#define MKB_ENTER(h)                                                        \
    if (!(h)) return MKB_ERR_BAD_ARG;                                       \
    mkb::DeviceGuard _guard((h)->device);                                   \
    if (!_guard.ok) return mkb::fail((h), MKB_ERR_CUDA, "cudaSetDevice(%d) failed", (h)->device)

// scope guard of every entry point that enqueues work on a caller's stream (see mkb_ctx::mtx)
struct StreamOrder {
    mkb_ctx *h;
    cudaStream_t st;
    std::unique_lock<std::recursive_mutex> lock;
    StreamOrder(mkb_ctx *h_, cudaStream_t st_) : h(h_), st(st_), lock(h_->mtx) {
        if (h->order_valid && h->order_stream != st) cudaStreamWaitEvent(st, h->order_ev, 0);
    }
    ~StreamOrder() {
        if (!h->order_ev && cudaEventCreateWithFlags(&h->order_ev, cudaEventDisableTiming) != cudaSuccess) return;
        if (cudaEventRecord(h->order_ev, st) == cudaSuccess) {
            h->order_stream = st;
            h->order_valid = true;
        }
    }
};
#define MKB_STREAM_ORDER(h, st) mkb::StreamOrder _order((h), (st))

#define MKB_LAUNCHED(h)                                                                                    \
    do {                                                                                                   \
        cudaError_t _e = cudaGetLastError();                                                               \
        if (_e != cudaSuccess)                                                                             \
            return mkb::fail((h), MKB_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), \
                             __FILE__, __LINE__);                                                          \
        (h)->launches++;                                                                                   \
    } while (0)

inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

}  // namespace mkb
