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
    S_TILE_TOTAL,   // occupancy warp kernel: halo atom count per block
    S_BLOCK_BASE,   // occupancy warp kernel: first block id of every grid
    S_K4_BALLOTS,   // contacts: hit masks of the count pass, reused by the fill pass
    S_BAND_BITMAP,  // occupancy run kernel: one bit per voxel whose gate decision is re-done in float64
    S_QUEUE,        // occupancy run kernel: block queue counter
    S_FIX_LIST,     // occupancy run kernel: voxels re-evaluated in float64 (count + list)
    S_BLK_ENT,      // occupancy run kernel: per-block candidate lists
    S_BLK_SEGS,     // occupancy run kernel: the (CTA, block) list segments reserved by the count pass
    S_ALIGN_PART,   // K14: per-(segment, frame) partial sums of the fit / RMSD
    S_ALIGN_REF,    // K14: the centred reference selection
    S_COORD_PART,   // K15: per-(frame chunk, atom, axis) partial frame sums
    S_SASA_REC,     // K17: gathered (x, y, z, R) records of a frame chunk
    S_SASA_SORTED,  // K17: the records sorted by cell bucket
    S_SASA_ITEM,    // K17: (bucket, slot) of every record
    S_SASA_SIDX,    // K17: environment index of every sorted record
    S_SASA_COUNT,   // K17: atoms per bucket
    S_SASA_START,   // K17: first sorted record of every bucket
    S_SASA_MAXR,    // K17: largest radius
    S_SASA_AREA,    // K17: per-atom areas before the group sums
    S_DSSP,         // K18: the per-frame arrays of one frame chunk, carved from one allocation
    S_TMSCORE_MASK, // K19: two cut-set bitmasks per resident thread
    S_MOMENT_TAB,   // K20: segment table, group offsets / totals and weights, uploaded per call
    S_MOMENT_PART,  // K20: per-(segment, frame) partial moment sums
    S_XYZ_COUNTS,   // K26: newlines (K28: atom records) per 32 KB segment
    S_XYZ_BASE,     // K26: number of the first newline (K28: atom record) of every segment
    S_XYZ_STARTS,   // K26: line starts (K28: atom record starts) of the staged frames
    S_XYZ_STATE,    // K26 / K28: the decode's running line (atom record) count
    S_BOND_MIN,     // K7: per-axis coordinate minimum (the reference's xyzmin) as order keys
    S_TMALIGN,      // K27: per-item traces, index lists and DP state of one item chunk
    S_BCIF_VAL,     // K31: two 32-bit value arrays of a column's decode or encode, used in turn
    S_BCIF_IDX,     // K31: int64 scans (value ranks, run starts, packed offsets)
    S_BCIF_TMP,     // K31: cub temp storage and the listed frames
    S_LMP_BITMAP,   // K32: one bit per (listed frame, atom row) of a decode: the ids seen
    S_LMP_LEN,      // K32: line lengths and their exclusive scan of an encode
    S_LMP_TMP,      // K32: cub temp storage of the encode's scan
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
    cudaEvent_t aux_ev[4] = {};  // band fork / join; block-index copy of the to-host route (issued / done)
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

// K14 fit record [16] float64: R (3x3 row-major), p_bar (3), q_bar (3), pad
__device__ __forceinline__ void fit_record_load(const double *r, double (&R)[9], double (&pb)[3], double (&qb)[3]) {
#pragma unroll
    for (int j = 0; j < 9; ++j) R[j] = r[j];
#pragma unroll
    for (int d = 0; d < 3; ++d) { pb[d] = r[9 + d]; qb[d] = r[12 + d]; }
}

// y = fl32(R (x - p_bar) + q_bar) evaluated in float64: the one definition of an aligned coordinate (K14 apply and the
// K15 coordinate / frame-sum / fluctuation kernels), so the in-place and the gathered results cannot drift apart
__device__ __forceinline__ void fit_transform(const double (&R)[9], const double (&pb)[3], const double (&qb)[3],
                                              float x0f, float x1f, float x2f, float (&y)[3]) {
    const double x0 = (double)x0f - pb[0], x1 = (double)x1f - pb[1], x2 = (double)x2f - pb[2];
#pragma unroll
    for (int d = 0; d < 3; ++d)
        y[d] = __double2float_rn(fma(R[3 * d + 2], x2, fma(R[3 * d + 1], x1, R[3 * d] * x0)) + qb[d]);
}

// fl(fl(fl(dx dx) + fl(dy dy)) + fl(dz dz)): the reference's float32 squared norm, the one definition every pair kernel
// compares and sums with
__device__ __forceinline__ float sq3(float dx, float dy, float dz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

}  // namespace mkb
