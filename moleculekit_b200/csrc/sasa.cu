// sasa.cu -- K17: Shrake-Rupley solvent-accessible surface area over a trajectory for sm_90a (H100).
//
// Replaces mdtraj's single-frame C++ loop (mdtraj/geometry/src/sasa.cpp, asa_frame) that moleculekit's MetricSasa calls
// once per frame.  Every decision is a float32 comparison evaluated with the reference's roundings (__fsub_rn /
// __fmul_rn / __fadd_rn, no contraction), and the area is a count of accessible points, so the result is bit-identical
// to the reference arithmetic whatever order the points and neighbours are visited in.
//
//   units       x_nm = fl(x / 10); R = radius + probe in nm, given per environment atom.
//   neighbours  j != i with d2 < fl(fl(R_i + R_j)^2), d2 = fl(fl(fl(dx dx) + fl(dy dy)) + fl(dz dz)), dx = fl(x_i - x_j).
//   points      p = fl(x_i + fl(R_i s)) per axis; buried when some neighbour k has |fl(p - x_k)|^2 (same sum) < fl(R_k R_k).
//   area        fl(fl(fl(c R_i) R_i) n_i), c = (float)(4 pi / N), n_i = accessible points; fl(area 100) in atom mode, or
//               fl(sum 100) of a group's areas added in order into a float32 zero.
//
// Per chunk of listed frames (bounded scratch, SA_CHUNK_BYTES):
//   gather     frame-major float4 (x_nm, y_nm, z_nm, R) records; each finite atom counts itself into a hashed cell
//              bucket of its frame (cells wider than 2 max R, index computed in float64, so +-1 cell holds every
//              neighbour; a hash collision only adds candidates, which the exact test rejects).
//   scan       cub exclusive sum of the bucket counts of the whole chunk; scatter the records bucket by bucket.
//   surface    one warp per (frame, query atom): the exact neighbour set of the 27 cells goes into a shared buffer as
//              (x, y, z, fl(R^2)); each lane owns SA_PTS sphere points per pass in registers with a mask of those not
//              yet buried, and the warp walks the buffer until no point of the pass is uncovered.  A neighbour list
//              longer than the buffer is walked in buffer-sized pieces, and gathered again for each later pass.
//   groups     one thread per (frame, group) adds the per-atom areas of the group in order (residue mode).
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "common.cuh"

namespace mkb {

constexpr int SA_WARPS = 8;
constexpr int SA_THREADS = 32 * SA_WARPS;
constexpr int SA_PTS = 8;                       // sphere points per lane per pass
constexpr int SA_PASS = 32 * SA_PTS;            // sphere points per pass
constexpr int SA_BUF = 128;                     // neighbour buffer entries per warp
constexpr double SA_CELL_CLAMP = 1073741824.0;  // |cell index| <= 2^30: clamping keeps adjacent cells adjacent
constexpr size_t SA_CHUNK_BYTES = size_t(256) << 20;
constexpr int SA_MAX_POINTS = 65536;

struct SasaArgs {
    const float *coords;
    long long fs;
    const unsigned *env;
    long long n_env;
    const float *radii;
    const unsigned *query;
    long long nq;
    const float *sphere;
    int npts;
    const unsigned *frames;
    float area_c;
    int hmask;                // buckets per frame - 1 (a power of two minus one)
};

struct SasaChunk {
    float4 *rec;              // [fc][n_env] gathered records
    int2 *item;               // [fc][n_env] (bucket or -1, slot in bucket)
    int *count;               // [fc][H] atoms per bucket
    int *start;               // [fc][H] first sorted entry of the bucket (chunk-wide)
    float4 *srec;             // sorted records
    int *sidx;                // environment index of each sorted record
    const float *maxr;        // largest radius
};

__device__ __forceinline__ double sa_width(const float *maxr) { return fmax(2.0 * (double)*maxr * (1.0 + 1e-5), 1e-6); }

__device__ __forceinline__ long long sa_cell(float x, double w) {
    return (long long)fmin(fmax(floor((double)x / w), -SA_CELL_CLAMP), SA_CELL_CLAMP);
}

__device__ __forceinline__ int sa_hash(long long cx, long long cy, long long cz, int hmask) {
    unsigned long long h = (unsigned long long)cx * 73856093ull ^ (unsigned long long)cy * 19349663ull ^
                           (unsigned long long)cz * 83492791ull;
    h ^= h >> 29;
    return (int)(h & (unsigned long long)hmask);
}

// fl(fl(fl(a.x b.x) + fl(a.y b.y)) + fl(a.z b.z)) of the difference a - b: SSE dpps with mask 0x71
__device__ __forceinline__ float sa_d2(float ax, float ay, float az, float bx, float by, float bz) {
    return sq3(__fsub_rn(ax, bx), __fsub_rn(ay, by), __fsub_rn(az, bz));
}

__global__ void sasa_maxr_kernel(const float *__restrict__ radii, long long n, float *__restrict__ maxr) {
    __shared__ float part[256];
    float m = 0.f;
    for (long long e = threadIdx.x; e < n; e += blockDim.x) m = fmaxf(m, radii[e]);
    part[threadIdx.x] = m;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) part[threadIdx.x] = fmaxf(part[threadIdx.x], part[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) *maxr = part[0];
}

// thread t = e * fc + kl (frame fastest: consecutive frames of one atom row are one coalesced read)
__global__ void sasa_gather_kernel(const SasaArgs A, long long k0, int fc, SasaChunk S) {
    const double w = sa_width(S.maxr);
    const long long total = (long long)fc * A.n_env, H = (long long)A.hmask + 1;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long e = t / fc, kl = t - e * fc, k = k0 + kl;
        const long long f = A.frames ? (long long)A.frames[k] : k;
        const float *src = A.coords + (long long)A.env[e] * 3 * A.fs + f;
        const float x = __fdiv_rn(__ldg(src), 10.f), y = __fdiv_rn(__ldg(src + A.fs), 10.f),
                    z = __fdiv_rn(__ldg(src + 2 * A.fs), 10.f);
        const long long r = kl * A.n_env + e;
        S.rec[r] = make_float4(x, y, z, __ldg(A.radii + e));
        int2 it = make_int2(-1, 0);
        if (isfinite(x) && isfinite(y) && isfinite(z)) {  // a non-finite atom has no neighbour relation: no cell
            it.x = sa_hash(sa_cell(x, w), sa_cell(y, w), sa_cell(z, w), A.hmask);
            it.y = atomicAdd(S.count + kl * H + it.x, 1);
        }
        S.item[r] = it;
    }
}

__global__ void sasa_scatter_kernel(const SasaArgs A, int fc, SasaChunk S) {
    const long long total = (long long)fc * A.n_env, H = (long long)A.hmask + 1;
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < total; r += (long long)gridDim.x * blockDim.x) {
        const int2 it = S.item[r];
        if (it.x < 0) continue;
        const long long kl = r / A.n_env;
        const int pos = S.start[kl * H + it.x] + it.y;
        S.srec[pos] = S.rec[r];
        S.sidx[pos] = (int)(r - kl * A.n_env);
    }
}

// clears the mask bits of the lane's points that neighbours buf[0, n) bury; stops once no lane has a point left
__device__ __forceinline__ void sa_walk(const float4 *buf, int n, const float (&px)[SA_PTS], const float (&py)[SA_PTS],
                                        const float (&pz)[SA_PTS], unsigned &mask) {
    for (int m = 0; m < n; ++m) {
        const float4 v = buf[m];
#pragma unroll
        for (int u = 0; u < SA_PTS; ++u)
            if (sa_d2(px[u], py[u], pz[u], v.x, v.y, v.z) < v.w) mask &= ~(1u << u);
        if (!__any_sync(0xffffffffu, mask)) break;
    }
}

// dst[kl * ld + q] = area of query q in chunk frame kl (nm^2, or Angstrom^2 with scale100)
__global__ void __launch_bounds__(SA_THREADS) sasa_surface_kernel(const SasaArgs A, long long k0, SasaChunk S,
                                                                  float *__restrict__ dst, long long ld, int scale100,
                                                                  unsigned long long *__restrict__ status) {
    __shared__ float4 sbuf[SA_WARPS][SA_BUF];
    const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
    const long long q = (long long)blockIdx.x * SA_WARPS + wi;
    if (q >= A.nq) return;  // whole warps only: no block-wide barrier follows
    float4 *buf = sbuf[wi];
    const long long kl = blockIdx.y, H = (long long)A.hmask + 1;
    const int i = (int)A.query[q];
    const float4 ri = S.rec[kl * A.n_env + i];
    const float Ri = ri.w;
    const bool finite = isfinite(ri.x) && isfinite(ri.y) && isfinite(ri.z);
    const double w = sa_width(S.maxr);
    const long long cx = finite ? sa_cell(ri.x, w) : 0, cy = finite ? sa_cell(ri.y, w) : 0,
                    cz = finite ? sa_cell(ri.z, w) : 0;
    const int *count = S.count + kl * H, *start = S.start + kl * H;
    const unsigned lt = (1u << lane) - 1u;
    const unsigned long long key = ((unsigned long long)(k0 + kl) << 32) | (unsigned long long)q;
    int accessible = 0, nbuf = 0;
    bool fits = false;
    for (int pass = 0; pass * SA_PASS < A.npts; ++pass) {
        float px[SA_PTS], py[SA_PTS], pz[SA_PTS];
        unsigned mask = 0;
#pragma unroll
        for (int u = 0; u < SA_PTS; ++u) {
            const int j = pass * SA_PASS + u * 32 + lane;
            px[u] = py[u] = pz[u] = 0.f;
            if (j < A.npts) {
                const float *s = A.sphere + 3 * j;
                px[u] = __fadd_rn(ri.x, __fmul_rn(Ri, __ldg(s)));
                py[u] = __fadd_rn(ri.y, __fmul_rn(Ri, __ldg(s + 1)));
                pz[u] = __fadd_rn(ri.z, __fmul_rn(Ri, __ldg(s + 2)));
                mask |= 1u << u;
            }
        }
        if (finite && fits) {
            sa_walk(buf, nbuf, px, py, pz, mask);
        } else if (finite) {
            // gather the neighbours again; the first pass reads every candidate (the coincidence check must see all of
            // them), later passes stop once every point of the pass is buried
            bool over = false, stop = false;
            nbuf = 0;
            for (int c = 0; c < 27 && !stop; ++c) {
                const int b = sa_hash(cx + c % 3 - 1, cy + (c / 3) % 3 - 1, cz + c / 9 - 1, A.hmask);
                const int s0 = start[b], n = count[b];
                for (int base = 0; base < n; base += 32) {
                    const int m = base + lane;
                    bool hit = false;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (m < n && S.sidx[s0 + m] != i) {
                        v = S.srec[s0 + m];
                        const float d2 = sa_d2(ri.x, ri.y, ri.z, v.x, v.y, v.z);
                        const float rc = __fadd_rn(Ri, v.w);
                        hit = d2 < __fmul_rn(rc, rc);
                        if (pass == 0 && d2 < 1e-10f) atomicMin(status, key);
                    }
                    const unsigned bal = __ballot_sync(0xffffffffu, hit);
                    if (hit) buf[nbuf + __popc(bal & lt)] = make_float4(v.x, v.y, v.z, __fmul_rn(v.w, v.w));
                    nbuf += __popc(bal);
                    if (nbuf > SA_BUF - 32) {
                        __syncwarp();
                        if (__any_sync(0xffffffffu, mask)) sa_walk(buf, nbuf, px, py, pz, mask);
                        __syncwarp();
                        over = true;
                        nbuf = 0;
                        if (pass > 0 && !__any_sync(0xffffffffu, mask)) { stop = true; break; }
                    }
                }
            }
            __syncwarp();
            if (nbuf > 0 && __any_sync(0xffffffffu, mask)) sa_walk(buf, nbuf, px, py, pz, mask);
            fits = !over;
        }
        accessible += __popc(mask);
    }
    const int n_i = __reduce_add_sync(0xffffffffu, accessible);
    if (lane == 0) {
        float a = __fmul_rn(__fmul_rn(__fmul_rn(A.area_c, Ri), Ri), (float)n_i);
        if (scale100) a = __fmul_rn(a, 100.f);
        dst[kl * ld + q] = a;
    }
}

__global__ void sasa_group_kernel(const float *__restrict__ areas, long long nq, const long long *__restrict__ goff,
                                  long long ng, int fc, float *__restrict__ out, long long ld) {
    const long long total = (long long)fc * ng;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long kl = t / ng, g = t - kl * ng;
        float s = 0.f;
        for (long long q = goff[g]; q < goff[g + 1]; ++q) s = __fadd_rn(s, areas[kl * nq + q]);
        out[kl * ld + g] = __fmul_rn(s, 100.f);
    }
}

inline long long sa_buckets(long long n_env) {
    long long H = 32;
    while (H < n_env) H <<= 1;
    return H;
}

// frames per chunk: scratch of one frame is its records, items, sorted records and indices, bucket counts and starts,
// and (with groups) the per-atom areas
inline long long sa_chunk_frames(long long n_env, long long nq, long long ng) {
    const long long H = sa_buckets(n_env);
    const long long per = n_env * (long long)(2 * sizeof(float4) + sizeof(int2) + sizeof(int)) + H * 2 * (long long)sizeof(int) +
                          (ng > 0 ? nq * (long long)sizeof(float) : 0);
    long long fc = std::max<long long>(1, (long long)SA_CHUNK_BYTES / per);
    fc = std::min<long long>(fc, 65535);
    return std::min<long long>(fc, std::max<long long>(1, ((1ll << 31) - 1) / std::max(n_env, H)));
}

}  // namespace mkb

using namespace mkb;

extern "C" int64_t mkb_sasa_chunk_frames(int64_t n_env, int64_t n_query, int64_t n_groups) {
    if (n_env < 1 || n_query < 0 || n_groups < 0) return 0;
    return sa_chunk_frames(n_env, n_query, n_groups);
}

extern "C" int mkb_sasa(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *env, int64_t n_env,
                        const float *radii, const uint32_t *query, int64_t n_query, const int64_t *group_offsets,
                        int64_t n_groups, const float *sphere, int32_t n_sphere, const uint32_t *frames, int64_t n_frames,
                        float *out, int64_t ld_out, int64_t *status) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (n_env < 1 || n_query < 1) return fail(h, MKB_ERR_BAD_ARG, "n_env and n_query must be >= 1");
    if (group_offsets && n_groups < 1) return fail(h, MKB_ERR_BAD_ARG, "n_groups must be >= 1 with group offsets");
    if (n_env > 0x7fffffffll || n_query > 0x7fffffffll) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_sphere < 1 || n_sphere > SA_MAX_POINTS)
        return fail(h, MKB_ERR_BAD_ARG, "n_sphere %d outside [1, %d]", (int)n_sphere, SA_MAX_POINTS);
    if (t->n_frames < 0 || (frames && n_frames < 0)) return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (!t->coords || !env || !radii || !query || !sphere || !status) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (((uintptr_t)status & 7) != 0) return fail(h, MKB_ERR_BAD_ARG, "status must be 8-byte aligned");
    if (t->frame_stride < t->n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const long long cols = group_offsets ? n_groups : n_query;
    if (ld_out < cols) return fail(h, MKB_ERR_BAD_ARG, "ld_out %lld < %lld output columns", (long long)ld_out, cols);
    const long long n = frames ? n_frames : t->n_frames;
    MKB_CUDA(h, cudaMemsetAsync(status, 0xff, sizeof(int64_t), st));
    if (n == 0) return MKB_OK;
    if (!out) return fail(h, MKB_ERR_BAD_ARG, "null out");
    const long long ng = group_offsets ? n_groups : 0;
    const long long H = sa_buckets(n_env), fc_max = sa_chunk_frames(n_env, n_query, ng);
    if (cdiv(n_query, SA_WARPS) >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many query atoms for one launch");

    SasaArgs A;
    A.coords = t->coords; A.fs = t->frame_stride;
    A.env = env; A.n_env = n_env; A.radii = radii;
    A.query = query; A.nq = n_query;
    A.sphere = sphere; A.npts = n_sphere;
    A.frames = frames;
    A.area_c = (float)(4.0 * 3.14159265358979323846 / (double)n_sphere);
    A.hmask = (int)(H - 1);

    const long long fcn = std::min(n, fc_max);
    SasaChunk S;
    float *maxr = nullptr, *areas = nullptr;
    void *tmp = nullptr;
    int rc;
    if ((rc = scratch_get(h, S_SASA_REC, (size_t)(fcn * n_env), &S.rec)) != MKB_OK) return rc;
    if ((rc = scratch_get(h, S_SASA_SORTED, (size_t)(fcn * n_env), &S.srec)) != MKB_OK) return rc;
    if ((rc = scratch_get(h, S_SASA_ITEM, (size_t)(fcn * n_env), &S.item)) != MKB_OK) return rc;
    if ((rc = scratch_get(h, S_SASA_SIDX, (size_t)(fcn * n_env), &S.sidx)) != MKB_OK) return rc;
    if ((rc = scratch_get(h, S_SASA_COUNT, (size_t)(fcn * H), &S.count)) != MKB_OK) return rc;
    if ((rc = scratch_get(h, S_SASA_START, (size_t)(fcn * H), &S.start)) != MKB_OK) return rc;
    if ((rc = scratch_get(h, S_SASA_MAXR, 1, &maxr)) != MKB_OK) return rc;
    if (ng && (rc = scratch_get(h, S_SASA_AREA, (size_t)(fcn * n_query), &areas)) != MKB_OK) return rc;
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, S.count, S.start, (int)(fcn * H), st));
    if ((rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp)) != MKB_OK) return rc;
    S.maxr = maxr;

    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    sasa_maxr_kernel<<<1, 256, 0, st>>>(radii, n_env, maxr);
    MKB_LAUNCHED(h);
    const int blocks = h->sm_count * 8;
    for (long long k0 = 0; k0 < n; k0 += fcn) {
        const int fc = (int)std::min(fcn, n - k0);
        MKB_CUDA(h, cudaMemsetAsync(S.count, 0, sizeof(int) * (size_t)(fc * H), st));
        const long long items = (long long)fc * n_env;
        const int gb = (int)std::min<long long>(cdiv(items, 256), blocks);
        sasa_gather_kernel<<<gb, 256, 0, st>>>(A, k0, fc, S);
        MKB_LAUNCHED(h);
        MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, S.count, S.start, (int)(fc * H), st));
        sasa_scatter_kernel<<<gb, 256, 0, st>>>(A, fc, S);
        MKB_LAUNCHED(h);
        const dim3 grid((unsigned)cdiv(n_query, SA_WARPS), (unsigned)fc);
        if (ng) {
            sasa_surface_kernel<<<grid, SA_THREADS, 0, st>>>(A, k0, S, areas, n_query, 0,
                                                             reinterpret_cast<unsigned long long *>(status));
            MKB_LAUNCHED(h);
            const int bb = (int)std::min<long long>(cdiv((long long)fc * ng, 256), blocks);
            sasa_group_kernel<<<bb, 256, 0, st>>>(areas, n_query, reinterpret_cast<const long long *>(group_offsets), ng, fc, out + k0 * ld_out, ld_out);
        } else {
            sasa_surface_kernel<<<grid, SA_THREADS, 0, st>>>(A, k0, S, out + k0 * ld_out, ld_out, 1,
                                                             reinterpret_cast<unsigned long long *>(status));
        }
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "sasa_surface_kernel";
    return MKB_OK;
}
