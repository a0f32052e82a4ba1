// bonds.cu -- K7 (SURVEY row a13, stretch): bond perception on a uniform non-periodic cell grid for sm_90a (H100).
//
// Replaces moleculekit/bondguesser.py:259-392 (bond_grid_search: Python dict binning + one Cython call per occupied
// box) and moleculekit/bondguesser_utils/bondguesser_utils.pyx:30-163 (half-shell neighbour table, _is_close,
// grid_bonds).  The reference's result is, as a SET, every atom pair that is not H-H with
// 0.001 <= d2 <= pairdist^2 and d2 <= (0.6 (r_i + r_j))^2, all in float32 with individually rounded operations; the
// cell grid only prunes the search.  Here: atoms are hashed into cells of edge pairdist(1+1e-5) (count -> scan ->
// order), one thread per atom visits the 27 neighbouring cells and keeps partners with a larger index, two passes
// (count, cub scan, fill).  Pairs come out as (i < j); the host wrapper sorts them into the canonical order the
// reference's own test compares in (calculateUniqueBonds).
#include <cub/device/device_scan.cuh>

#include <cmath>

#include "common.cuh"

namespace mkb {

__device__ __forceinline__ unsigned bond_hash(int cx, int cy, int cz, unsigned hmask) {
    const unsigned long long h = (unsigned long long)(long long)cx * 73856093ull ^
                                 (unsigned long long)(long long)cy * 19349663ull ^
                                 (unsigned long long)(long long)cz * 83492791ull;
    return (unsigned)((h ^ (h >> 23)) & hmask);
}

// cell index in float64: with cells 1e-5 wider than the cutoff, two atoms within the cutoff along an axis are at most one
// cell apart for any coordinate magnitude a float can resolve
__device__ __forceinline__ int cell_of(float x, double inv_w) { return (int)floor((double)x * inv_w); }

__global__ void bond_bin_kernel(const float *__restrict__ coords, long long n, double inv_w, unsigned hmask,
                                unsigned *__restrict__ item_bucket, unsigned *__restrict__ item_slot,
                                unsigned *__restrict__ bucket_count) {
    const long long a = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (a >= n) return;
    const unsigned b = bond_hash(cell_of(coords[3 * a], inv_w), cell_of(coords[3 * a + 1], inv_w),
                                 cell_of(coords[3 * a + 2], inv_w), hmask);
    item_bucket[a] = b;
    item_slot[a] = atomicAdd(&bucket_count[b], 1u);
}

__global__ void bond_order_kernel(long long n, const unsigned *__restrict__ item_bucket,
                                  const unsigned *__restrict__ item_slot, const unsigned *__restrict__ bucket_start,
                                  unsigned *__restrict__ order) {
    const long long a = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (a >= n) return;
    order[bucket_start[item_bucket[a]] + item_slot[a]] = (unsigned)a;
}

// bondguesser_utils.pyx:89-115 (_is_close), float32 ops individually rounded, double only where the reference
// promotes (the 0.001 and 0.6 literals)
__device__ __forceinline__ bool bonded(const float *__restrict__ c, const float *__restrict__ radii,
                                       const unsigned *__restrict__ is_h, long long i, long long j, float cutoff2) {
    if (is_h[i] && is_h[j]) return false;
    const float dx = __fsub_rn(c[3 * i], c[3 * j]), dy = __fsub_rn(c[3 * i + 1], c[3 * j + 1]),
                dz = __fsub_rn(c[3 * i + 2], c[3 * j + 2]);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    if (d2 > cutoff2 || (double)d2 < 0.001) return false;
    const float cut = (float)(0.6 * (double)__fadd_rn(radii[i], radii[j]));
    return !(d2 > __fmul_rn(cut, cut));
}

template <bool FILL>
__global__ void bond_pairs_kernel(const float *__restrict__ coords, const float *__restrict__ radii,
                                  const unsigned *__restrict__ is_h, long long n, double inv_w, float cutoff2,
                                  unsigned hmask, const unsigned *__restrict__ bucket_start,
                                  const unsigned *__restrict__ order, long long *__restrict__ row_counts,
                                  const long long *__restrict__ row_offsets, unsigned *__restrict__ pairs) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int cx = cell_of(coords[3 * i], inv_w), cy = cell_of(coords[3 * i + 1], inv_w),
              cz = cell_of(coords[3 * i + 2], inv_w);
    long long cnt = 0, pos = FILL ? row_offsets[i] : 0;
    for (int k = 0; k < 27; ++k) {
        const int nx = cx + k / 9 - 1, ny = cy + (k / 3) % 3 - 1, nz = cz + k % 3 - 1;
        const unsigned b = bond_hash(nx, ny, nz, hmask);
        for (unsigned t = bucket_start[b]; t < bucket_start[b + 1]; ++t) {
            const long long j = order[t];
            if (j <= i) continue;  // each unordered pair once, as (min, max)
            // a bucket may hold atoms of other cells with the same hash: only count true members of this cell
            if (cell_of(coords[3 * j], inv_w) != nx || cell_of(coords[3 * j + 1], inv_w) != ny ||
                cell_of(coords[3 * j + 2], inv_w) != nz)
                continue;
            if (bonded(coords, radii, is_h, i, j, cutoff2)) {
                if (FILL) { pairs[2 * pos] = (unsigned)i; pairs[2 * pos + 1] = (unsigned)j; ++pos; }
                else ++cnt;
            }
        }
    }
    if (!FILL) row_counts[i] = cnt;
}

__global__ void bond_set_last_zero(long long *p, long long n) {
    if (threadIdx.x == 0 && blockIdx.x == 0) p[n] = 0;
}

struct BondGrid {
    unsigned hmask;
    double inv_w;
    float cutoff2;
    unsigned *bstart, *order;
};

static int bond_build(mkb_ctx *h, cudaStream_t st, const float *coords, int64_t n, float pairdist, BondGrid *g) {
    unsigned nb = 1024;
    while ((long long)nb < 2 * n && nb < (1u << 22)) nb <<= 1;
    g->hmask = nb - 1;
    g->inv_w = 1.0 / ((double)pairdist * 1.00001);  // cells slightly wider than the cutoff: +-1 cell is always enough
    g->cutoff2 = pairdist * pairdist;         // pyx:136: float product
    unsigned *ibucket, *islot, *bcount;
    int rc;
    const size_t na = (size_t)std::max<long long>(n, 1);
    if ((rc = scratch_get(h, S_ITEM_CELL, na, &ibucket))) return rc;
    if ((rc = scratch_get(h, S_ITEM_SLOT, na, &islot))) return rc;
    if ((rc = scratch_get(h, S_CELL_COUNT, (size_t)nb + 1, &bcount))) return rc;
    if ((rc = scratch_get(h, S_PT_BUCKET, (size_t)nb + 1, &g->bstart))) return rc;
    if ((rc = scratch_get(h, S_PT_ORDER, na, &g->order))) return rc;
    MKB_CUDA(h, cudaMemsetAsync(bcount, 0, sizeof(unsigned) * ((size_t)nb + 1), st));
    const unsigned gr = (unsigned)cdiv(n, 256);
    bond_bin_kernel<<<gr, 256, 0, st>>>(coords, n, g->inv_w, g->hmask, ibucket, islot, bcount);
    MKB_LAUNCHED(h);
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, bcount, g->bstart, (int)nb + 1, st));
    void *tmp = nullptr;
    if ((rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp))) return rc;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, bcount, g->bstart, (int)nb + 1, st));
    h->launches++;
    bond_order_kernel<<<gr, 256, 0, st>>>(n, ibucket, islot, g->bstart, g->order);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

static int bond_args(mkb_ctx *h, const float *coords, const float *radii, const uint32_t *is_h, int64_t n,
                     float pairdist) {
    if (n < 0) return fail(h, MKB_ERR_BAD_ARG, "negative atom count");
    if (n >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "n_atoms must be < 2^31");
    if (!(pairdist > 0.f) || !std::isfinite(pairdist)) return fail(h, MKB_ERR_BAD_ARG, "pairdist must be positive and finite");
    if (n > 0 && (!coords || !radii || !is_h)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    return MKB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// K10 (SURVEY 8f row 3): `within` / `exwithin` selections.  Replaces within_distance
// (moleculekit/atomselect_utils/atomselect_utils.pyx:612-653), a brute-force n1 x n2 loop with a TODO for a cell list.
// The source atoms (sel2) are hashed into cells of edge cutoff(1+1e-5) with the K7 machinery; one thread per query atom
// visits its 27 cells and stops at the first partner with ((dx*dx) + dy*dy) + dz*dz < cutoff*cutoff -- float32, each
// operation rounded, strict '<' (pyx:628,647-650).  The answer is an OR, so the visiting order does not matter.
// ---------------------------------------------------------------------------------------------------------
__global__ void within_gather_kernel(const float *__restrict__ coords, const unsigned *__restrict__ sel, long long n,
                                     float *__restrict__ out) {
    const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long a = sel[k];
    out[3 * k] = coords[3 * a]; out[3 * k + 1] = coords[3 * a + 1]; out[3 * k + 2] = coords[3 * a + 2];
}

__global__ void within_kernel(const float *__restrict__ coords, const unsigned *__restrict__ sel1, long long n1,
                              const float *__restrict__ src, double inv_w, float sq_cutoff, unsigned hmask,
                              const unsigned *__restrict__ bucket_start, const unsigned *__restrict__ order,
                              unsigned char *__restrict__ results) {
    const long long ii = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (ii >= n1) return;
    const long long i = sel1 ? (long long)sel1[ii] : ii;
    const float x = coords[3 * i], y = coords[3 * i + 1], z = coords[3 * i + 2];
    if (!(x == x && y == y && z == z)) return;  // a NaN coordinate is never within anything (and has no cell)
    const int cx = cell_of(x, inv_w), cy = cell_of(y, inv_w), cz = cell_of(z, inv_w);
    for (int k = 0; k < 27; ++k) {
        const int nx = cx + k / 9 - 1, ny = cy + (k / 3) % 3 - 1, nz = cz + k % 3 - 1;
        const unsigned b = bond_hash(nx, ny, nz, hmask);
        for (unsigned t = bucket_start[b]; t < bucket_start[b + 1]; ++t) {
            const float *s = src + 3ll * order[t];
            // atoms of other cells sharing the bucket are simply tested as well: any true hit is a valid answer
            const float dx = __fsub_rn(x, s[0]), dy = __fsub_rn(y, s[1]), dz = __fsub_rn(z, s[2]);
            const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            if (d2 < sq_cutoff) { results[ii] = 1; return; }
        }
    }
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_within_distance(mkb_handle_t h, void *stream, const float *coords, int64_t n_atoms,
                                   const uint32_t *sel1, int64_t n1, const uint32_t *sel2, int64_t n2, float cutoff,
                                   uint8_t *results) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_atoms < 0 || n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_atoms >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "n_atoms must be < 2^31");
    if (cutoff != cutoff || std::isinf(cutoff)) return fail(h, MKB_ERR_BAD_ARG, "cutoff must be finite");
    if (n1 == 0 || n2 == 0 || n_atoms == 0) return MKB_OK;
    if (!coords || !sel2 || !results) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (!sel1 && n1 != n_atoms) return fail(h, MKB_ERR_BAD_ARG, "sel1 == NULL means all atoms: n1 must equal n_atoms");
    // cutoff*cutoff is what the reference compares with (pyx:628), so a negative cutoff behaves like its magnitude;
    // cutoff == 0 can match nothing (d2 < 0 is impossible)
    const float sq = cutoff * cutoff;
    if (!(sq > 0.f)) return MKB_OK;
    float *src;
    int rc;
    if ((rc = scratch_get(h, S_SORT_PX, (size_t)n2 * 3, &src))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    within_gather_kernel<<<(unsigned)cdiv(n2, 256), 256, 0, st>>>(coords, sel2, n2, src);
    MKB_LAUNCHED(h);
    BondGrid g;
    if ((rc = bond_build(h, st, src, n2, std::fabs(cutoff), &g))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    within_kernel<<<(unsigned)cdiv(n1, 128), 128, 0, st>>>(coords, sel1, n1, src, g.inv_w, sq, g.hmask, g.bstart, g.order,
                                                           results);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_bonds_count(mkb_handle_t h, void *stream, const float *coords, const float *radii,
                               const uint32_t *is_hydrogen, int64_t n, float pairdist, int64_t *row_offsets,
                               int64_t *total_pairs) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    int rc = bond_args(h, coords, radii, is_hydrogen, n, pairdist);
    if (rc) return rc;
    if (!row_offsets || !total_pairs) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets/total_pairs");
    long long *counts;
    if ((rc = scratch_get(h, S_ROWCNT, (size_t)n + 1, &counts))) return rc;
    if (n > 0) {
        BondGrid g;
        if ((rc = bond_build(h, st, coords, n, pairdist, &g))) return rc;
        bond_pairs_kernel<false><<<(unsigned)cdiv(n, 128), 128, 0, st>>>(coords, radii, is_hydrogen, n, g.inv_w,
                                                                         g.cutoff2, g.hmask, g.bstart, g.order, counts,
                                                                         nullptr, nullptr);
        MKB_LAUNCHED(h);
    }
    bond_set_last_zero<<<1, 32, 0, st>>>(counts, n);
    MKB_LAUNCHED(h);
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, (long long *)row_offsets, (int)n + 1, st));
    void *tmp = nullptr;
    if ((rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp))) return rc;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, (long long *)row_offsets, (int)n + 1, st));
    h->launches++;
    long long total = 0;
    MKB_CUDA(h, cudaMemcpyAsync(&total, row_offsets + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    *total_pairs = total;
    return MKB_OK;
}

extern "C" int mkb_bonds_fill(mkb_handle_t h, void *stream, const float *coords, const float *radii,
                              const uint32_t *is_hydrogen, int64_t n, float pairdist, const int64_t *row_offsets,
                              uint32_t *pairs) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    int rc = bond_args(h, coords, radii, is_hydrogen, n, pairdist);
    if (rc) return rc;
    if (n == 0) return MKB_OK;
    if (!row_offsets || !pairs) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets/pairs");
    BondGrid g;
    if ((rc = bond_build(h, st, coords, n, pairdist, &g))) return rc;
    bond_pairs_kernel<true><<<(unsigned)cdiv(n, 128), 128, 0, st>>>(coords, radii, is_hydrogen, n, g.inv_w, g.cutoff2,
                                                                    g.hmask, g.bstart, g.order, nullptr,
                                                                    (const long long *)row_offsets, pairs);
    MKB_LAUNCHED(h);
    return MKB_OK;
}
