// occupancy.cu -- K1/K1b/K2: voxel occupancy for sm_90a (H100).
//
// Replaces moleculekit/occupancy_utils/occupancy_utils.pyx:34-61 (calculate_occupancy) and the grid-centre
// materialisation of moleculekit/tools/voxeldescriptors.py:125-132,197-248 on the device.
//
// Algorithm (not a translation of the reference's atoms x centres double loop):
//   value(c,h) = max_a [ d2 < 25 ] (1 - exp(-(sigma_ah^2/d2)^6)).   f(q) = 1 - exp(-q^6) is monotone in
//   q = sigma^2/d2, so the max over atoms commutes with f: the hot loop only tracks max q per voxel-channel and the
//   transcendental runs ONCE per voxel-channel in the epilogue.
//   K1  three fill kernels; occupancy_grid_batch_impl picks one per call from the input alone:
//       occ_fill_runs_kernel (occ_runs.cuh, fed by its own block lists K2'): 8 channels, no accumulate, 16-byte aligned
//         output, cutoff <= 40 voxels -- the default;
//       occ_fill8v_kernel: the other calls with <= 8 channels and a cutoff <= 14 voxels, one warp per 2x4x8 block;
//       occ_fill_kernel<CP>: everything else (9..32 channels, finer grids, or the 15..40-voxel cutoffs the run kernel
//         does not serve), described below.
//   K2  bin atoms of every grid of the batch into cells (count -> cub scan -> scatter): 4 voxels for occ_fill8v_kernel,
//       8 otherwise; positions kept as float64 voxel coordinates p' = (x - origin)/voxelsize.
//   occ_fill_kernel: one CTA (512 threads) per 8x8x8-voxel tile: gather the tile's halo atoms from <= (R+1)^2 contiguous
//       cell rows into shared memory as float positions RELATIVE TO THE TILE CORNER (|rel| < 32, so fp32 keeps ~5e-7
//       voxel absolute accuracy wherever the molecule sits), then each warp owns a 2x4x4 voxel block, culls the list
//       against its block with one ballot per 32 atoms and accumulates max q in registers (8 channels = 8 FMNMX).
//       Pairs whose d2 falls within 4e-6 (relative) of the 5 A gate are re-evaluated in float64 with the reference's
//       exact operation order, so the discontinuity at the gate is reproduced bit-for-bit.
//       Output: coalesced 32-byte (8-channel) streaming stores, 4 lanes = one 128-byte line.
// HBM-bound gather-accumulate: no tensor cores (max of a transcendental is not a contraction).
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <cuda.h>  // CUtensorMap (types only; the encoder is looked up through the runtime, libcuda is not linked)

#include <cfloat>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <thread>
#include <utility>
#include <vector>

#include "common.cuh"

namespace mkb {

constexpr int TILE = 8;
constexpr float TILE_C = 0.5f * (TILE - 1);  // tile-frame origin: centre of the 8-voxel tile
constexpr int FILL_THREADS = 512;
constexpr int LIST_CAP = 1536;
constexpr double CUTOFF_A = 5.0;      // occupancy_utils.pyx:53: dist2 < 25
constexpr float GATE_BAND = 4e-6f;    // relative half-width of the float64 re-check band around the gate

struct GridDev {
    double origin[3];
    double vs;
    double inv_vs;
    int dims[3];
    int tiles[3];
    int cells[3];
    int cutv;    // halo in voxels: ceil(5 / vs)
    int rcells;  // neighbour reach in cells: (TILE - 1 + 2 cutv) / TILE
    float cut2v, cut2v_lo, cut2v_hi;  // (5/vs)^2 in voxel units and the re-check band
    int cell;    // cell edge in voxels (8 for the tile kernels, 4 for the warp-per-block kernel)
    long long atom_begin, atom_end, out_offset;
    long long item_base, tile_base, cell_base;
    long long vox_base;  // first voxel of this grid in the dense batch order (gate-band bitmap of the run kernel)
    long long blk_base;  // run kernel: first 4x4x8 block of this grid (compact records); its lists are per 8x8x8 tile (tile_base)
};

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// 1 - exp(-q^6), q = sigma^2/d2  (== 1 - exp(-(sigma/r)^12), occupancy_utils.pyx:57-60), relative error ~1e-6.
__device__ __forceinline__ float occ_value(float q) {
    const float q2 = q * q;
    const float q3 = q2 * q;
    const float t = q3 * q3;
    // small t: -expm1(-t) by Taylor (avoids the cancellation that costs 0.4 relative error in naive fp32)
    // below t = 0.25 the t^6 / 5040 term is 4.8e-8 of the value: under half a float ulp
    float s = fmaf(t, -1.0f / 720.0f, 1.0f / 120.0f);
    s = fmaf(t, s, -1.0f / 24.0f);
    s = fmaf(t, s, 1.0f / 6.0f);
    s = fmaf(t, s, -0.5f);
    s = fmaf(t, s, 1.0f);
    s = s * t;
    const float b = 1.0f - ex2_approx(t * -1.4426950408889634f);
    return t < 0.25f ? s : b;
}

__device__ __forceinline__ int find_grid_item(const GridDev *g, int B, long long v) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (g[mid].item_base <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---------------------------------------------------------------------------------------------------------
// K2a: per (grid, atom) item -> cell id + slot inside the cell (atomic counter).
// ---------------------------------------------------------------------------------------------------------
__global__ void occ_bin_kernel(const float *__restrict__ coords, const GridDev *__restrict__ grids, int B,
                               long long n_items, int *__restrict__ item_cell, unsigned *__restrict__ item_slot,
                               unsigned *__restrict__ cell_count) {
    const long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (it >= n_items) return;
    const int b = find_grid_item(grids, B, it);
    const GridDev &g = grids[b];
    const long long a = g.atom_begin + (it - g.item_base);
    int c[3];
    bool live = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double p = ((double)coords[3 * a + d] - g.origin[d]) * g.inv_vs;
        // atoms farther than the 5 A halo from the grid cannot touch any voxel (NaN fails both tests)
        live = live && (p >= -(double)g.cutv) && (p <= (double)(g.dims[d] - 1 + g.cutv));
        int ci = live ? (int)floor((p + (double)g.cutv) / (double)g.cell) : 0;
        c[d] = min(max(ci, 0), g.cells[d] - 1);
    }
    if (!live) {
        item_cell[it] = -1;
        return;
    }
    const int cid = (c[0] * g.cells[1] + c[1]) * g.cells[2] + c[2];
    item_cell[it] = cid;
    item_slot[it] = atomicAdd(&cell_count[g.cell_base + cid], 1u);
}

// ---------------------------------------------------------------------------------------------------------
// K2b: scatter items into cell order (SoA).  sigma handling: the common case (moleculekit's boolean channels times
// one vdW radius, voxeldescriptors.py:332-335) has ONE distinct non-zero sigma per atom -> one s2 and a channel
// bit mask.  Atoms with several distinct sigmas are flagged (bit 31 of src) and take a per-channel path in K1.
// ---------------------------------------------------------------------------------------------------------
__global__ void occ_scatter_kernel(const float *__restrict__ coords, const double *__restrict__ sigmas,
                                   const double *__restrict__ radii, const unsigned *__restrict__ chanmask, int C,
                                   const GridDev *__restrict__ grids, int B, long long n_items,
                                   const int *__restrict__ item_cell, const unsigned *__restrict__ item_slot,
                                   const unsigned *__restrict__ cell_start, float4 *__restrict__ rec_pos,
                                   uint4 *__restrict__ rec_tag) {
    const long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (it >= n_items) return;
    const int cid = item_cell[it];
    if (cid < 0) return;
    const int b = find_grid_item(grids, B, it);
    const GridDev &g = grids[b];
    const long long a = g.atom_begin + (it - g.item_base);
    const unsigned dst = cell_start[g.cell_base + cid] + item_slot[it];
    // position relative to the atom's own cell origin (float64 subtraction, one rounding to float: |rel| < cell <= 8 voxels,
    // absolute error <= 2.4e-7 voxel); the cell coordinates travel in the tag so a tile can rebase exactly.
    const int cz = cid % g.cells[2], cxy = cid / g.cells[2], cy = cxy % g.cells[1], cx = cxy / g.cells[1];
    const int cc[3] = {cx, cy, cz};
    float rel[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double pv = ((double)coords[3 * a + d] - g.origin[d]) * g.inv_vs;
        rel[d] = (float)(pv - (double)(cc[d] * g.cell - g.cutv));
    }
    double first = 0.0;
    unsigned m = 0;
    bool multi = false;
    if (sigmas) {
        const double *sg = sigmas + a * C;
        for (int h = 0; h < C; ++h) {
            const double s = sg[h];
            if (s == 0.0 || s != s) continue;  // sigma == 0 skipped (pyx:56); NaN never wins the max (pyx:61)
            if (m == 0) { first = s; m = 1u << h; }
            else if (s == first) m |= 1u << h;
            else multi = true;
        }
    } else {
        // device-side channel assembly (voxeldescriptors.py:332-335): sigmas[a, h] = radii[a] * float(mask bit h), i.e.
        // one radius on the channels of the mask; a zero / NaN radius switches the atom off exactly as above
        const double r = radii[a];
        const unsigned mm = chanmask[a] & (C >= 32 ? 0xffffffffu : ((1u << C) - 1u));
        if (mm && !(r == 0.0 || r != r)) { first = r; m = mm; }
    }
    const double sv = first * g.inv_vs;  // sigma in voxel units
    rec_pos[dst] = make_float4(rel[0], rel[1], rel[2], m ? fmaxf((float)(sv * sv), FLT_MIN) : 0.0f);
    // tag.w: 1/|sigma| (voxel units) for the run kernel, which tracks min d2/sigma^2 on coordinates pre-scaled by it
    const float sw = m ? (float)(1.0 / fabs(sv)) : 0.0f;
    rec_tag[dst] = make_uint4(m, (unsigned)a | (multi ? 0x80000000u : 0u), (unsigned)cx | ((unsigned)cy << 10) | ((unsigned)cz << 20),
                              __float_as_uint(sw));
}

// ---------------------------------------------------------------------------------------------------------
// K1: tile fill.
// ---------------------------------------------------------------------------------------------------------
struct FillParams {
    const GridDev *grids;
    int B, C;
    const float4 *rec_pos;  // cell-sorted atoms: x, y, z relative to the cell origin (voxels), sigma^2 (voxels^2)
    const uint4 *rec_tag;   // channel mask, atom row | multi-sigma flag << 31, packed cell coordinates
    const unsigned *cell_start;
    const float *coords;
    const double *sigmas;
    float *out;
    unsigned flags;
    int vec_ok;
    int cmajor;     // MKB_OCC_LAYOUT_CXYZ: grid b is stored [C][nx][ny][nz] (channel-major) instead of [nx][ny][nz][C]
    int txp_shift;  // warp kernel launch: blockIdx.z = (grid << txp_shift) | block_x
    // warp kernel, uniform launches: descriptor of the chunk's first grid + per-grid strides
    GridDev u;
    long long u_out_stride, u_cell_stride, u_block_base, u_block_stride;
    unsigned u_band_bits;  // width of the gate re-check band, precomputed for uniform launches (constant bank operand)
};

// float64 re-evaluation of the gate with the reference's exact operations (pyx:49-53; centres as built by
// voxeldescriptors.py:125-132,245: fl(fl(i*vs) + origin)).
__device__ __noinline__ bool exact_gate(const GridDev *g, const float *coords, unsigned a, int ix, int iy, int iz) {
    const double cx = __dadd_rn(__dmul_rn((double)ix, g->vs), g->origin[0]);
    const double cy = __dadd_rn(__dmul_rn((double)iy, g->vs), g->origin[1]);
    const double cz = __dadd_rn(__dmul_rn((double)iz, g->vs), g->origin[2]);
    const double dx = (double)coords[3ll * a + 0] - cx;
    const double dy = (double)coords[3ll * a + 1] - cy;
    const double dz = (double)coords[3ll * a + 2] - cz;
    const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    return d2 < CUTOFF_A * CUTOFF_A;
}

constexpr int MAX_ROWS = FILL_THREADS;  // cell rows feeding one tile: (R+1)^2, R = (TILE-1+2*cutv)/TILE

__device__ __forceinline__ float4 lds_f4(unsigned addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ unsigned lds_u16(unsigned addr) {
    unsigned short v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ unsigned lds_u32(unsigned addr) {
    unsigned v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// grid = (max tiles per grid, B): blockIdx.y is the grid (molecule / pocket), blockIdx.x its tile.
template <int CP>
__global__ void __launch_bounds__(FILL_THREADS, (CP <= 8 ? 2 : 1)) occ_fill_kernel(const FillParams p) {
    __shared__ float4 s_ent[LIST_CAP];    // x, y, z relative to the tile corner (voxel units), w = sigma^2 (voxel units)
    __shared__ unsigned s_mask[LIST_CAP]; // channel bits of the atom's single sigma; 0 = several sigmas (slow path)
    __shared__ unsigned s_src[LIST_CAP];  // atom row (exact gate / multi-sigma path)
    __shared__ unsigned s_rpos[MAX_ROWS]; // first sorted atom of each cell row
    __shared__ unsigned s_rbase[MAX_ROWS + 1];  // exclusive prefix of the row lengths
    __shared__ GridDev s_g;
    __shared__ int s_cnt;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const GridDev *gg = p.grids + blockIdx.y;
    {
        const int ntiles = __ldg(&gg->tiles[0]) * __ldg(&gg->tiles[1]) * __ldg(&gg->tiles[2]);
        if ((int)blockIdx.x >= ntiles) return;  // ragged batch: this grid has fewer tiles than the largest one
    }
    if (tid < (int)(sizeof(GridDev) / 4)) reinterpret_cast<unsigned *>(&s_g)[tid] = reinterpret_cast<const unsigned *>(gg)[tid];
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    const GridDev &g = s_g;

    const int nx = g.dims[0], ny = g.dims[1], nz = g.dims[2];
    const int tzN = g.tiles[2], tyN = g.tiles[1];
    const int local = blockIdx.x;
    const int tz = local % tzN, txy = local / tzN, ty = txy % tyN, tx = txy / tyN;

    // cell rows feeding this tile: cells [tx, tx+R] x [ty, ty+R], each a contiguous z-run [tz, tz+R]
    const int R = g.rcells;
    const int cN1 = g.cells[1], cN2 = g.cells[2];
    const int cx1 = min(tx + R, g.cells[0] - 1), cy1 = min(ty + R, cN1 - 1), cz1 = min(tz + R, cN2 - 1);
    const int ncy = cy1 - ty + 1;
    const int nrows = (cx1 - tx + 1) * ncy;
    if (tid < nrows) {
        const int rx = tid / ncy, ry = tid - rx * ncy;
        const long long cb = g.cell_base + ((long long)(tx + rx) * cN1 + (ty + ry)) * cN2;
        const unsigned a = __ldg(p.cell_start + cb + tz), e = __ldg(p.cell_start + cb + cz1 + 1);
        s_rpos[tid] = a;
        s_rbase[tid + 1] = e - a;
    }
    if (tid == 0) s_rbase[0] = 0;
    __syncthreads();
    if (warp == 0) {  // inclusive scan of the row lengths (nrows <= 512: 16 chunks of 32 at most)
        unsigned carry = 0;
        for (int c0 = 0; c0 < nrows; c0 += 32) {
            const int r = c0 + lane;
            unsigned v = (r < nrows) ? s_rbase[r + 1] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v += t;
            }
            if (r < nrows) s_rbase[r + 1] = v + carry;
            carry += __shfl_sync(0xffffffffu, v, 31);
        }
    }
    __syncthreads();
    const unsigned total = s_rbase[nrows];

    // warp -> 2x4x4 voxel block of the tile, lane -> voxel (z fastest so 4 lanes cover one 128-byte output line)
    const int bx = warp >> 2, by = (warp >> 1) & 1, bz = warp & 1;
    const int vx = bx * 2 + (lane >> 4), vy = by * 4 + ((lane >> 2) & 3), vz = bz * 4 + (lane & 3);
    const int C = p.C;

    float acc[CP];
#pragma unroll
    for (int h = 0; h < CP; ++h) acc[h] = 0.0f;
    bool touched = false;

    if (total != 0) {
        // tile frame: origin at the tile CENTRE (voxel 3.5), so |coordinate| <= 3.5 + cutv and fp32 spacing is finest
        const float fvx = (float)vx - TILE_C, fvy = (float)vy - TILE_C, fvz = (float)vz - TILE_C;
        const float bcx = (float)(bx * 2) - TILE_C, bcy = (float)(by * 4) - TILE_C, bcz = (float)(bz * 4) - TILE_C;
        const float cut2v = g.cut2v, cut_hi = g.cut2v_hi, band = g.cut2v_hi - g.cut2v;
        const int cshift_x = tx * TILE + g.cutv, cshift_y = ty * TILE + g.cutv, cshift_z = tz * TILE + g.cutv;
        // 32-bit shared-window addresses taken ONCE (volatile: ptxas otherwise rebuilds them from SR_CgaCtaId per use)
        unsigned ent_sa, mask_sa;
        asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(ent_sa) : "l"(s_ent));
        asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(mask_sa) : "l"(s_mask));

        for (unsigned c0 = 0; c0 < total; c0 += LIST_CAP) {  // one pass unless > LIST_CAP atoms sit in the halo
            if (c0) {
                __syncthreads();  // previous pass fully consumed
                if (tid == 0) s_cnt = 0;
                __syncthreads();
            }
            const unsigned c1 = min(total, c0 + (unsigned)LIST_CAP);
            // ---- gather: every thread takes atoms k = c0 + tid, + 512, ... of the concatenated cell rows
            for (unsigned k0 = c0; k0 < c1; k0 += FILL_THREADS) {
                const unsigned k = k0 + tid;
                bool pass = false;
                float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
                unsigned m = 0, sr = 0;
                if (k < c1) {
                    int lo = 0, hi = nrows - 1;  // row with rbase[row] <= k < rbase[row + 1]
                    while (lo < hi) {
                        const int mid = (lo + hi + 1) >> 1;
                        if (s_rbase[mid] <= k) lo = mid; else hi = mid - 1;
                    }
                    const unsigned i = s_rpos[lo] + (k - s_rbase[lo]);
                    e = __ldg(p.rec_pos + i);
                    const uint4 tg = __ldg(p.rec_tag + i);
                    m = tg.x;
                    sr = tg.y;
                    e.x += (float)((int)(tg.z & 1023u) * TILE - cshift_x) - TILE_C;  // exact: small integers
                    e.y += (float)((int)((tg.z >> 10) & 1023u) * TILE - cshift_y) - TILE_C;
                    e.z += (float)((int)(tg.z >> 20) * TILE - cshift_z) - TILE_C;
                    const float ddx = fmaxf(fabsf(e.x) - TILE_C, 0.f);
                    const float ddy = fmaxf(fabsf(e.y) - TILE_C, 0.f);
                    const float ddz = fmaxf(fabsf(e.z) - TILE_C, 0.f);
                    pass = (m != 0) && (ddx * ddx + ddy * ddy + ddz * ddz <= cut_hi);
                    if (sr & 0x80000000u) m = 0;  // several distinct sigmas: per-channel path
                }
                const unsigned bal = __ballot_sync(0xffffffffu, pass);
                if (bal) {
                    int base = 0;
                    if (lane == 0) base = atomicAdd(&s_cnt, __popc(bal));
                    base = __shfl_sync(0xffffffffu, base, 0);
                    if (pass) {
                        const int slot = base + __popc(bal & ((1u << lane) - 1u));
                        s_ent[slot] = e;
                        s_mask[slot] = m;
                        s_src[slot] = sr & 0x7fffffffu;
                    }
                }
            }
            __syncthreads();
            const int n = s_cnt;

            // ---- consume: each warp culls the list against its 2x4x4 block, then all lanes evaluate the survivors
            for (int j0 = 0; j0 < n; j0 += 32) {
                const int j = j0 + lane;
                bool hit = false;
                if (j < n) {
                    const float4 e = s_ent[j];
                    const float rx = e.x - bcx, ry = e.y - bcy, rz = e.z - bcz;
                    const float ddx = fmaxf(fmaxf(-rx, rx - 1.f), 0.f);
                    const float ddy = fmaxf(fmaxf(-ry, ry - 3.f), 0.f);
                    const float ddz = fmaxf(fmaxf(-rz, rz - 3.f), 0.f);
                    hit = (ddx * ddx + ddy * ddy + ddz * ddz) <= cut_hi;
                }
                unsigned bal = __ballot_sync(0xffffffffu, hit);
                touched = touched || (bal != 0);
                while (bal) {
                    const int jj = j0 + __ffs(bal) - 1;
                    bal &= bal - 1;
                    const float4 e = lds_f4(ent_sa + jj * 16);
                    const unsigned cm = lds_u32(mask_sa + jj * 4);
                    const float dx = e.x - fvx, dy = e.y - fvy, dz = e.z - fvz;
                    const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
                    const float r = rcp_approx(d2);
                    float gate = (d2 < cut2v) ? 1.0f : 0.0f;
                    if (fabsf(d2 - cut2v) <= band)  // within 4e-6 of the gate: decide exactly like the reference
                        gate = exact_gate(&g, p.coords, s_src[jj], tx * TILE + vx, ty * TILE + vy, tz * TILE + vz) ? 1.0f : 0.0f;
                    const bool in = gate != 0.0f;
                    const float q = in ? e.w * r : 0.0f;  // sigma^2/d2; +inf at d2 == 0 -> value 1
                    if (cm != 0) {
#pragma unroll
                        for (int h = 0; h < CP; ++h)
                            if (cm & (1u << h)) acc[h] = fmaxf(acc[h], q);
                    } else {
                        // several distinct sigmas on this atom: per-channel q (user-supplied float channels)
                        const double *sg = p.sigmas + (long long)s_src[jj] * C;
                        const double ivs = g.inv_vs;
                        const float rr = in ? r : 0.0f;
#pragma unroll
                        for (int h = 0; h < CP; ++h) {
                            if (h < C) {
                                const double s = sg[h] * ivs;
                                const float sq = (s == 0.0 || s != s) ? 0.0f : fmaxf((float)(s * s), FLT_MIN);
                                acc[h] = fmaxf(acc[h], sq * rr);  // 0*inf = NaN is dropped by fmaxf
                            }
                        }
                    }
                }
            }
        }
    }

    // ---- epilogue: one transcendental per voxel-channel, streaming 32-byte stores
    const int ix = tx * TILE + vx, iy = ty * TILE + vy, iz = tz * TILE + vz;
    if (ix < nx && iy < ny && iz < nz) {
        const long long vox = ((long long)ix * ny + iy) * nz + iz;
        const long long cs = p.cmajor ? (long long)nx * ny * nz : 1;  // channel stride; voxel stride is C or 1
        float *const o = p.out + g.out_offset * C + vox * (p.cmajor ? 1 : C);
        float v[CP];
        if (touched) {
#pragma unroll
            for (int h = 0; h < CP; ++h) v[h] = occ_value(acc[h]);
        } else {
#pragma unroll
            for (int h = 0; h < CP; ++h) v[h] = 0.0f;
        }
        if (p.flags & MKB_OCC_ACCUMULATE) {
#pragma unroll
            for (int h = 0; h < CP; ++h)
                if (h < C) { const float old = o[h * cs]; v[h] = (acc[h] > 0.0f && v[h] > old) ? v[h] : old; }  // pyx:61 `value > old`
        }
        if (CP == 8 && p.vec_ok) {
            __stcs(reinterpret_cast<float4 *>(o), make_float4(v[0], v[1], v[2], v[3]));
            __stcs(reinterpret_cast<float4 *>(o) + 1, make_float4(v[4], v[5], v[6], v[7]));
        } else {
#pragma unroll
            for (int h = 0; h < CP; ++h)
                if (h < C) o[h * cs] = v[h];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// K1 v6 (C <= 8 channels, cutoff <= 14 voxels, calls the run kernel does not serve): no CTA-level synchronisation.
//   Each warp owns one 2x4x8 voxel block end to end: it gathers the block's own halo from 4-voxel cells (<= 64 contiguous
//   cell rows) into its private shared-memory list, splits it into eight 2x2x2 sub-block lists (sy in 0..1, sz in 0..3,
//   four lanes each) and runs them in lock-step; empty blocks retire after one halo count.  A lane owns the x-pair of
//   voxels (0, y, z) and (1, y, z).  Against one voxel per lane on 2x4x4 blocks:
//     * one halo gather (cell rows are contiguous along z, so doubling the block along z adds ~20 % scanned atoms, not
//       100 %), one row set-up, one prologue per 64 voxels instead of per 32;
//     * a candidate is loaded once for two voxels that share dy, dz and the channel mask: 39 instructions per candidate
//       for two pairs instead of 30 for one, while each 2x2x2 sub-block keeps its own list (same 47 % hit rate);
//     * two independent dependency chains per lane (ILP) stand in for the halved number of resident warps.
// ---------------------------------------------------------------------------------------------------------
constexpr int V_CELL = 4;     // cell edge of the binning used with this kernel
constexpr int V_ROWS = 64;    // cell rows per block: (Rx+1)(Ry+1) <= 64 up to a 14-voxel cutoff
constexpr int V_BZ = 8;       // block extent along z
// capacity sweep (ms per 256 pockets): 128/96 1.864, 160/96 1.858, 224/96 1.841, 192/128 1.814, 224/128 1.825, 256/128 1.850
constexpr int V_PCAP = 192;   // block candidates per round
constexpr int V_QCAP = 128;   // sub-block candidates per round
constexpr int V_QSTRIDE = V_QCAP + 2;  // + one sentinel slot for the software-pipelined loop
constexpr int V_WARPS = 1;    // warps (= blocks) per CTA. A CTA holds its registers until its slowest warp retires
constexpr int V_MIN_CTAS = 7; // 72 registers; at 8 CTAs (64 registers) the kernel spills
constexpr float GATE_SCALE = 1.2676506002282294e30f;  // 2^100

__global__ void occ_block_total_v_kernel(const GridDev *__restrict__ grids, const unsigned *__restrict__ cell_start,
                                         const long long *__restrict__ block_base, unsigned *__restrict__ block_total) {
    const GridDev &g = grids[blockIdx.y];
    const int nbx = (g.dims[0] + 1) / 2, nby = (g.dims[1] + 3) / 4, nbz = (g.dims[2] + V_BZ - 1) / V_BZ;
    const int local = blockIdx.x * blockDim.x + threadIdx.x;
    if (local >= nbx * nby * nbz) return;
    const int bzi = local % nbz, bxy = local / nbz, byi = bxy % nby, bxi = bxy / nby;
    const int cutv = g.cutv, cN1 = g.cells[1], cN2 = g.cells[2];
    const int cx0 = (bxi * 2) / V_CELL, cx1 = min((bxi * 2 + 1 + 2 * cutv) / V_CELL, g.cells[0] - 1);
    const int cy0 = byi, cy1 = min((byi * 4 + 3 + 2 * cutv) / V_CELL, cN1 - 1);
    const int cz0 = bzi * (V_BZ / V_CELL), cz1 = min((bzi * V_BZ + V_BZ - 1 + 2 * cutv) / V_CELL, cN2 - 1);
    unsigned total = 0;
    for (int cx = cx0; cx <= cx1; ++cx)
        for (int cy = cy0; cy <= cy1; ++cy) {
            const long long cb = g.cell_base + ((long long)cx * cN1 + cy) * cN2;
            total += cell_start[cb + cz1 + 1] - cell_start[cb + cz0];
        }
    block_total[block_base[blockIdx.y] + local] = total;
}

// UNIFORM: every grid of the launch has the same shape (the batched-pockets case): shape constants come from the
// kernel parameters (constant bank) instead of a chain of dependent global loads -- an empty block then waits for ONE
// load (its halo count) before it can retire.
#define WG(field) (UNIFORM ? p.u.field : __ldg(&gg->field))
template <bool UNIFORM>
__global__ void __launch_bounds__(V_WARPS * 32, V_MIN_CTAS * 4 / V_WARPS)
occ_fill8v_kernel(const FillParams p, const long long *__restrict__ block_base, const unsigned *__restrict__ block_total) {
    __shared__ float4 s_pent[V_WARPS][V_PCAP + 1];    // block candidates: x, y, z in the block frame, sigma^2 (+ sentinel)
    __shared__ unsigned s_pmask[V_WARPS][V_PCAP + 1];  // channel mask; 0 = several sigmas
    __shared__ unsigned s_psrc[V_WARPS][V_PCAP];
    __shared__ unsigned s_rpos[V_WARPS][V_ROWS];
    __shared__ unsigned s_rbase[V_WARPS][V_ROWS + 1];
    __shared__ unsigned short s_qidx[V_WARPS][8][V_QSTRIDE];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int byi = blockIdx.y, bxi = blockIdx.z & ((1 << p.txp_shift) - 1);
    const int gi = blockIdx.z >> p.txp_shift;
    const GridDev *gg = p.grids + gi;
    const int nx = WG(dims[0]), ny = WG(dims[1]), nz = WG(dims[2]);
    const long long out_offset = UNIFORM ? p.u.out_offset + (long long)gi * p.u_out_stride : __ldg(&gg->out_offset);
    if (bxi * 2 >= nx || byi * 4 >= ny) return;  // padding of the launch grid / ragged batch
    const int C = p.C;
    const long long cs = p.cmajor ? (long long)nx * ny * nz : 1;  // channel stride; voxel stride is C or 1
    const int vstride = p.cmajor ? 1 : C;
    const int bzi = blockIdx.x * V_WARPS + warp;
    if (bzi * V_BZ >= nz) return;

    // ---- empty block (no atom within reach): stream 64 x 32 B of zeros and retire
    {
        const int nby = (ny + 3) >> 2, nbz = (nz + V_BZ - 1) / V_BZ;
        const long long bb = UNIFORM ? p.u_block_base + (long long)gi * p.u_block_stride : __ldg(block_base + gi);
        const unsigned tot = __ldg(block_total + bb + ((long long)bxi * nby + byi) * nbz + bzi);
        if (tot == 0 && !(p.flags & MKB_OCC_ACCUMULATE)) {
            const int iy = byi * 4 + (lane >> 3), iz = bzi * V_BZ + (lane & 7);  // 8 lanes = one 256-byte row
            if (iy < ny && iz < nz) {
#pragma unroll
                for (int v = 0; v < 2; ++v) {
                    const int ix = bxi * 2 + v;
                    if (ix < nx) {
                        float *d = p.out + out_offset * C + (((long long)ix * ny + iy) * nz + iz) * vstride;
                        if (p.vec_ok) {
                            const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
                            __stcs(reinterpret_cast<float4 *>(d), z4);
                            __stcs(reinterpret_cast<float4 *>(d) + 1, z4);
                        } else {
                            for (int h = 0; h < C; ++h) __stcs(d + h * cs, 0.f);
                        }
                    }
                }
            }
            return;
        }
    }

    // ---- cell rows of this block's halo (V_CELL = 4): rows run along z
    const int cutv = WG(cutv);
    const int cN1 = WG(cells[1]), cN2 = WG(cells[2]);
    const int cx0 = (bxi * 2) / V_CELL, cx1 = min((bxi * 2 + 1 + 2 * cutv) / V_CELL, WG(cells[0]) - 1);
    const int cy0 = byi, cy1 = min((byi * 4 + 3 + 2 * cutv) / V_CELL, cN1 - 1);
    const int cz0 = bzi * (V_BZ / V_CELL), cz1 = min((bzi * V_BZ + V_BZ - 1 + 2 * cutv) / V_CELL, cN2 - 1);
    const int ncy = cy1 - cy0 + 1;
    const int nrows = (cx1 - cx0 + 1) * ncy;  // <= V_ROWS checked on the host
    unsigned *const rpos = s_rpos[warp], *const rbase = s_rbase[warp];
    const long long cell_base = UNIFORM ? p.u.cell_base + (long long)gi * p.u_cell_stride : __ldg(&gg->cell_base);
    const float inv_ncy = 1.0f / (float)ncy;
    const float cut_hi_row = WG(cut2v_hi);
    unsigned carry = 0;
    for (int r0 = 0; r0 < nrows; r0 += 32) {  // row lengths + inclusive scan, 32 rows per step
        const int r = r0 + lane;
        unsigned v = 0;
        if (r < nrows) {
            const int rx = (int)(((float)r + 0.5f) * inv_ncy), ry = r - rx * ncy;  // exact for small r
            const long long cb = cell_base + ((long long)(cx0 + rx) * cN1 + (cy0 + ry)) * cN2;
            const unsigned a = __ldg(p.cell_start + cb + cz0);
            v = __ldg(p.cell_start + cb + cz1 + 1) - a;
            rpos[r] = a;
            // corner rows: the cell column [c*4 - cutv, c*4 + 4 - cutv) is further than the cutoff from the block's
            // x/y extent -> none of its atoms can pass the cull below, skip the row
            const int lox = (cx0 + rx) * V_CELL - cutv, loy = (cy0 + ry) * V_CELL - cutv;
            const int gx = max(max(lox - (bxi * 2 + 1), bxi * 2 - (lox + V_CELL)), 0);
            const int gy = max(max(loy - (byi * 4 + 3), byi * 4 - (loy + V_CELL)), 0);
            if ((float)(gx * gx + gy * gy) > cut_hi_row) v = 0;
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += t;
        }
        if (r < nrows) rbase[r + 1] = v + carry;
        carry += __shfl_sync(0xffffffffu, v, 31);
    }
    const unsigned total = carry;

    // lane -> sub-block s = (sy, sz) and position (ty, tz) in it; the lane's two voxels are x = 0 and x = 1
    const int s = lane >> 2, t4 = lane & 3;
    const int ly = (s >> 2) * 2 + (t4 >> 1), lz = (s & 3) * 2 + (t4 & 1);
    const int ix0 = bxi * 2, iy = byi * 4 + ly, iz = bzi * V_BZ + lz;
    const bool in_yz = iy < ny && iz < nz;
    const bool inside0 = in_yz && ix0 < nx, inside1 = in_yz && ix0 + 1 < nx;

    float acc0[8], acc1[8];
#pragma unroll
    for (int h = 0; h < 8; ++h) acc0[h] = acc1[h] = 0.0f;
    bool touched = false;

    if (total != 0) {
        if (lane == 0) {
            rbase[0] = 0;
            s_pent[warp][V_PCAP] = make_float4(1e18f, 1e18f, 1e18f, 0.0f);  // sentinel: never inside the gate
            s_pmask[warp][V_PCAP] = 1u;
        }
        __syncwarp();
        const float cut_lo = WG(cut2v_lo), cut_hi = WG(cut2v_hi);
        const unsigned band_bits = UNIFORM ? p.u_band_bits : __float_as_uint(cut_hi - cut_lo);
        const float fvy = (float)ly - 1.5f, fvz = (float)lz - 3.5f;  // block frame: origin at the block centre
        const int sx = bxi * 2 + cutv, sy = byi * 4 + cutv, sz = bzi * V_BZ + cutv;
        float4 *const pent = s_pent[warp];
        unsigned *const pmask = s_pmask[warp], *const psrc = s_psrc[warp];
        unsigned short *const wq = s_qidx[warp][0];
        unsigned short *const my_q = s_qidx[warp][s];
        unsigned ent_sa, mask_sa, q_sa;
        asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(ent_sa) : "l"(pent));
        asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(mask_sa) : "l"(pmask));
        asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(q_sa) : "l"(my_q));

        int np = 0;
        int row = 0;  // row of this lane's current atom: k only grows, so the row pointer only advances
        for (unsigned k0 = 0; k0 < total; k0 += 32) {
            // ---- gather 32 atoms of the concatenated cell rows, keep those within reach of the block
            {
                const unsigned k = min(k0 + lane, total - 1);
                while (rbase[row + 1] <= k) ++row;  // rbase[nrows] == total > k: terminates
                const unsigned i = rpos[row] + (k - rbase[row]);
                float4 e = __ldg(p.rec_pos + i);
                const uint4 tg = __ldg(p.rec_tag + i);
                e.x += (float)((int)(tg.z & 1023u) * V_CELL - sx) - 0.5f;  // exact: small integers and halves
                e.y += (float)((int)((tg.z >> 10) & 1023u) * V_CELL - sy) - 1.5f;
                e.z += (float)((int)(tg.z >> 20) * V_CELL - sz) - 3.5f;
                const float ddx = fmaxf(fabsf(e.x) - 0.5f, 0.f);
                const float ddy = fmaxf(fabsf(e.y) - 1.5f, 0.f);
                const float ddz = fmaxf(fabsf(e.z) - 3.5f, 0.f);
                const bool pass = (k0 + lane < total) & (tg.x != 0) & (fmaf(ddz, ddz, fmaf(ddy, ddy, ddx * ddx)) <= cut_hi);
                const unsigned bal = __ballot_sync(0xffffffffu, pass);
                if (pass) {
                    const int slot = np + __popc(bal & ((1u << lane) - 1u));
                    pent[slot] = e;
                    pmask[slot] = (tg.y & 0x80000000u) ? 0u : tg.x;
                    psrc[slot] = tg.y & 0x7fffffffu;
                }
                np += __popc(bal);
            }
            if (np <= V_PCAP - 32 && k0 + 32 < total) continue;
            if (np == 0) continue;
            touched = true;
            __syncwarp();
            // ---- block list -> eight 2x2x2 sub-block lists, evaluated in lock-step
            int cq[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) cq[u] = 0;
            for (int j0 = 0; j0 < np; j0 += 32) {
                const int j = j0 + lane;
                const bool live = j < np;
                const unsigned idx = min(j, np - 1);
                bool hit[8], multi;
                {
                    const float4 e = lds_f4(ent_sa + idx * 16);
                    const float ddx = fmaxf(fabsf(e.x) - 0.5f, 0.f);
                    const float y0 = fmaxf(fabsf(e.y + 1.f) - 0.5f, 0.f), y1 = fmaxf(fabsf(e.y - 1.f) - 0.5f, 0.f);
                    const float xx = ddx * ddx;
                    const float a0 = fmaf(y0, y0, xx), a1 = fmaf(y1, y1, xx);
                    multi = live & (lds_u32(mask_sa + idx * 4) == 0);
                    const bool ok = live & !multi;
#pragma unroll
                    for (int zz = 0; zz < 4; ++zz) {  // sub-block centres along z: -3, -1, +1, +3
                        const float zd = fmaxf(fabsf(e.z - (float)(2 * zz - 3)) - 0.5f, 0.f);
                        const float z2 = zd * zd;
                        hit[zz] = ok & (a0 + z2 <= cut_hi);      // s = sy*4 + sz
                        hit[4 + zz] = ok & (a1 + z2 <= cut_hi);
                    }
                }
                // atoms carrying several distinct sigmas (user float channels): whole-warp per-channel path
                for (unsigned bm = __ballot_sync(0xffffffffu, multi); bm; bm &= bm - 1) {
                    const int jj = j0 + __ffs(bm) - 1;
                    const float4 e = pent[jj];
                    const float dy = e.y - fvy, dz = e.z - fvz;
                    const float s2 = fmaf(dz, dz, dy * dy);
                    const double *sg = p.sigmas + (long long)psrc[jj] * C;
                    const double ivs = WG(inv_vs);
#pragma unroll
                    for (int v = 0; v < 2; ++v) {
                        const float dx = e.x - ((float)v - 0.5f);
                        const float d2 = fmaf(dx, dx, s2);
                        bool in = d2 < cut_lo;
                        if (!in && d2 < cut_hi) in = exact_gate(gg, p.coords, psrc[jj], ix0 + v, iy, iz);
                        const float rr = in ? rcp_approx(d2) : 0.0f;
#pragma unroll
                        for (int h = 0; h < 8; ++h) {
                            if (h < C) {
                                const double sv = sg[h] * ivs;
                                const float sq = (sv == 0.0 || sv != sv) ? 0.0f : fmaxf((float)(sv * sv), FLT_MIN);
                                if (v == 0) acc0[h] = fmaxf(acc0[h], sq * rr);  // 0*inf = NaN is dropped by fmaxf
                                else acc1[h] = fmaxf(acc1[h], sq * rr);
                            }
                        }
                    }
                }
                const unsigned lt = (1u << lane) - 1u;
                int nmax = 0;
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const unsigned b = __ballot_sync(0xffffffffu, hit[u]);
                    if (hit[u]) wq[u * V_QSTRIDE + cq[u] + __popc(b & lt)] = (unsigned short)idx;
                    cq[u] += __popc(b);
                    nmax = max(nmax, cq[u]);
                }
                if (j0 + 32 < np && nmax <= V_QCAP - 32) continue;
                // pad the shorter lists with the sentinel, then run all eight in lock-step
                int mine = cq[0];
#pragma unroll
                for (int u = 1; u < 8; ++u) mine = (s == u) ? cq[u] : mine;
                for (int c = mine + t4; c <= nmax; c += 4) my_q[c] = (unsigned short)V_PCAP;  // incl. slot nmax (prefetch)
                __syncwarp();
                auto candidate = [&](unsigned q_addr) {
                    const unsigned jj = lds_u16(q_addr);
                    const float4 e = lds_f4(ent_sa + jj * 16);
                    const unsigned cm = lds_u32(mask_sa + jj * 4);
                    const float dy = e.y - fvy, dz = e.z - fvz;
                    const float s2 = fmaf(dz, dz, dy * dy);
                    const float dx0 = e.x + 0.5f, dx1 = e.x - 0.5f;
                    const float d20 = fmaf(dx0, dx0, s2), d21 = fmaf(dx1, dx1, s2);
                    const float qf0 = e.w * rcp_approx(d20), qf1 = e.w * rcp_approx(d21);  // +inf at d2 == 0 -> value 1
                    // exact 0/1 gate on the FMA pipe: sat(2^100 (cut_lo - d2)) -- the difference is shared with the band test
                    const float t0 = d20 - cut_lo, t1 = d21 - cut_lo;
                    float qv0 = qf0 * __saturatef(t0 * -GATE_SCALE);
                    float qv1 = qf1 * __saturatef(t1 * -GATE_SCALE);
                    // within 4e-6 of the gate: decide like the reference (float64, its operation order)
                    const bool n0 = __float_as_uint(t0) < band_bits, n1 = __float_as_uint(t1) < band_bits;
                    if (n0 | n1) {
                        if (n0 && exact_gate(gg, p.coords, psrc[jj], ix0, iy, iz)) qv0 = qf0;
                        if (n1 && exact_gate(gg, p.coords, psrc[jj], ix0 + 1, iy, iz)) qv1 = qf1;
                    }
#pragma unroll
                    for (int h = 0; h < 8; ++h)
                        if (cm & (1u << h)) { acc0[h] = fmaxf(acc0[h], qv0); acc1[h] = fmaxf(acc1[h], qv1); }
                };
                for (unsigned qa = q_sa, qe = q_sa + 2 * nmax; qa < qe; qa += 2) candidate(qa);
                __syncwarp();
#pragma unroll
                for (int u = 0; u < 8; ++u) cq[u] = 0;
            }
            np = 0;
            __syncwarp();
        }
    }

    // ---- epilogue: one transcendental per non-zero voxel-channel (a channel that is zero across the warp -- metals,
    // charged groups -- skips it), 32-byte streaming stores (8 lanes = one 256-byte row)
    float val0[8], val1[8];
#pragma unroll
    for (int h = 0; h < 8; ++h) {
        val0[h] = val1[h] = 0.0f;
        if (touched && __any_sync(0xffffffffu, (acc0[h] != 0.0f) | (acc1[h] != 0.0f))) {
            val0[h] = occ_value(acc0[h]);
            val1[h] = occ_value(acc1[h]);
        }
    }
#pragma unroll
    for (int v = 0; v < 2; ++v) {
        if (v == 0 ? inside0 : inside1) {
            float val[8];
#pragma unroll
            for (int h = 0; h < 8; ++h) val[h] = v == 0 ? val0[h] : val1[h];
            float *const oo = p.out + out_offset * C + (((long long)(ix0 + v) * ny + iy) * nz + iz) * vstride;
            if (p.flags & MKB_OCC_ACCUMULATE) {
#pragma unroll
                for (int h = 0; h < 8; ++h)
                    if (h < C) {
                        const float old = oo[h * cs], q = v == 0 ? acc0[h] : acc1[h];
                        val[h] = (q > 0.0f && val[h] > old) ? val[h] : old;
                    }
            }
            if (p.vec_ok) {
                __stcs(reinterpret_cast<float4 *>(oo), make_float4(val[0], val[1], val[2], val[3]));
                __stcs(reinterpret_cast<float4 *>(oo) + 1, make_float4(val[4], val[5], val[6], val[7]));
            } else if (p.cmajor) {
#pragma unroll
                for (int h = 0; h < 8; ++h)
                    if (h < C) __stcs(oo + h * cs, val[h]);
            } else {
#pragma unroll
                for (int h = 0; h < 8; ++h)
                    if (h < C) oo[h] = val[h];
            }
        }
    }
    __syncwarp();  // no data hazard left; without it ptxas schedules the measured kernel differently
}
#undef WG

// ---------------------------------------------------------------------------------------------------------
// K1b: arbitrary centres.  Atoms hashed into 5 A cells (count -> scan -> order); one thread per centre visits the
// 27 neighbouring buckets.  Distances in float64 exactly as the reference (pyx:49-53), so the gate is exact.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned cell_hash(long long cx, long long cy, long long cz, unsigned hmask) {
    const unsigned long long h = (unsigned long long)cx * 73856093ull ^ (unsigned long long)cy * 19349663ull ^
                                 (unsigned long long)cz * 83492791ull;
    return (unsigned)((h ^ (h >> 23)) & hmask);
}

constexpr double PT_LIMIT = 1e12;  // beyond this nothing can be within 5 A in float32 coordinates that matter

__global__ void pt_bin_kernel(const float *__restrict__ coords, long long n, unsigned hmask,
                              int *__restrict__ item_bucket, unsigned *__restrict__ item_slot,
                              unsigned *__restrict__ bucket_count) {
    const long long a = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (a >= n) return;
    const double x = coords[3 * a], y = coords[3 * a + 1], z = coords[3 * a + 2];
    if (!(fabs(x) < PT_LIMIT && fabs(y) < PT_LIMIT && fabs(z) < PT_LIMIT)) { item_bucket[a] = -1; return; }
    const unsigned bkt = cell_hash((long long)floor(x * (1.0 / CUTOFF_A)), (long long)floor(y * (1.0 / CUTOFF_A)),
                                   (long long)floor(z * (1.0 / CUTOFF_A)), hmask);
    item_bucket[a] = (int)bkt;
    item_slot[a] = atomicAdd(&bucket_count[bkt], 1u);
}

__global__ void pt_order_kernel(long long n, const int *__restrict__ item_bucket, const unsigned *__restrict__ item_slot,
                                const unsigned *__restrict__ bucket_start, unsigned *__restrict__ order) {
    const long long a = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (a >= n) return;
    const int b = item_bucket[a];
    if (b < 0) return;
    order[bucket_start[b] + item_slot[a]] = (unsigned)a;
}

// Below SIGMA_EXACT the reference's own float64 result, 1 - exp(-x^12), is quantised to multiples of 2^-53 (exactly 0
// for x^12 < 2^-54): at d -> 5 A and sigma = 0.7 A, x^12 = (0.14)^12 = 5.7e-11, so the quantisation is already 1e-6 of
// the value, and it grows as sigma^-12 below that.  A float32 evaluation of the exact function cannot reproduce it; the
// points kernel evaluates such channels with the reference's float64 operations instead (s2 < 0 marks them); the grid
// entry points zero them for the grid kernels and run this kernel on the grid centres (occupancy_utils.py).  Bit parity
// with the reference there also needs the device's double exp to round like glibc's where x^12 is small and exp(-x^12)
// lands within a few ulp of 1: not guaranteed by either library, it holds on every case of
// tests/test_occupancy_contract_gpu.py::test_sigma_sweep.  The extra branch and the exact[] array cost every points call;
// that cost is not measured by bench.py (grid workloads only).
constexpr double SIGMA_EXACT = 0.7;

__global__ void pt_sigma_kernel(const double *__restrict__ sigmas, long long n, float *__restrict__ s2) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double s = sigmas[i];
    s2[i] = (s == 0.0 || s != s) ? 0.0f : (fabs(s) < SIGMA_EXACT ? -1.0f : fmaxf((float)(s * s), FLT_MIN));
}

template <int CP>
__global__ void __launch_bounds__(128) occ_points_kernel(const double *__restrict__ centers, long long M,
                                                         const float *__restrict__ coords,
                                                         const float *__restrict__ s2, const double *__restrict__ sigmas,
                                                         int C, unsigned hmask,
                                                         const unsigned *__restrict__ bucket_start,
                                                         const unsigned *__restrict__ order, float *__restrict__ out,
                                                         unsigned flags) {
    const long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (m >= M) return;
    const double cx = centers[3 * m], cy = centers[3 * m + 1], cz = centers[3 * m + 2];
    float acc[CP];
    float exact[CP];  // max of the float64 values of the sigma < SIGMA_EXACT channels; -1: no such atom reached
#pragma unroll
    for (int h = 0; h < CP; ++h) { acc[h] = 0.0f; exact[h] = -1.0f; }
    if (fabs(cx) < PT_LIMIT && fabs(cy) < PT_LIMIT && fabs(cz) < PT_LIMIT) {
        const long long kx = (long long)floor(cx * (1.0 / CUTOFF_A)), ky = (long long)floor(cy * (1.0 / CUTOFF_A)),
                        kz = (long long)floor(cz * (1.0 / CUTOFF_A));
        for (int n = 0; n < 27; ++n) {
            const unsigned bkt = cell_hash(kx + (n / 9) - 1, ky + ((n / 3) % 3) - 1, kz + (n % 3) - 1, hmask);
            const unsigned s = bucket_start[bkt], e = bucket_start[bkt + 1];
            for (unsigned i = s; i < e; ++i) {
                const unsigned a = order[i];
                const double dx = (double)coords[3ll * a + 0] - cx;
                const double dy = (double)coords[3ll * a + 1] - cy;
                const double dz = (double)coords[3ll * a + 2] - cz;
                const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                if (d2 < CUTOFF_A * CUTOFF_A) {
                    const float r = rcp_approx((float)d2);
                    const float *sa = s2 + (long long)a * C;
#pragma unroll
                    for (int h = 0; h < CP; ++h) {
                        if (h < C) {
                            const float s = sa[h];
                            if (s >= 0.0f) {
                                acc[h] = fmaxf(acc[h], s * r);  // A^2/A^2: same q as the grid path
                            } else {  // pyx:57-60 in the reference's order and precision
                                const double x = sigmas[(long long)a * C + h] / sqrt(d2);
                                const double x3 = (x * x) * x;
                                const double x12 = ((x3 * x3) * x3) * x3;
                                exact[h] = fmaxf(exact[h], (float)(1.0 - exp(-x12)));
                            }
                        }
                    }
                }
            }
        }
    }
    float *o = out + m * C;
#pragma unroll
    for (int h = 0; h < CP; ++h) {
        if (h < C) {
            const float v = fmaxf(occ_value(acc[h]), exact[h]);
            // accumulate: only a voxel-channel some atom with a non-zero sigma reached is updated (pyx:56-61)
            const bool reached = acc[h] > 0.0f || exact[h] >= 0.0f;
            if (flags & MKB_OCC_ACCUMULATE) { const float old = o[h]; o[h] = (reached && v > old) ? v : old; }
            else o[h] = v;
        }
    }
}

}  // namespace mkb
#include "occ_runs.cuh"

// 4-D tiled tensor map over a uniform dense batch: [grid][x][y][z * 8 channels] float32, box = one 4 x 4 x 8-voxel block.
// Returns false when the encoder is unavailable or rejects the layout (the caller keeps the row copies).
static bool occ_make_tmap(CUtensorMap *tm, float *base, int nx, int ny, int nz, long long n_grids, long long grid_stride_vox) {
    typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static encode_fn enc = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
            enc = (encode_fn)fn;
        else
            (void)cudaGetLastError();
    });
    if (!enc || ((uintptr_t)base & 15u)) return false;
    const cuuint64_t dims[4] = {(cuuint64_t)nz * 8, (cuuint64_t)ny, (cuuint64_t)nx, (cuuint64_t)n_grids};
    const cuuint64_t strides[3] = {(cuuint64_t)nz * 32, (cuuint64_t)ny * nz * 32, (cuuint64_t)grid_stride_vox * 32};  // bytes, dims 1..3
    const cuuint32_t box[4] = {mkb::R_BZ * 8, 4, 4, 1}, estr[4] = {1, 1, 1, 1};
    for (int i = 0; i < 3; ++i)
        if (strides[i] >= (1ull << 40)) return false;
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
namespace mkb {

static int scan_u32(mkb_ctx *h, cudaStream_t st, unsigned *in, unsigned *out, long long n) {
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, in, out, (int)n, st));
    void *tmp = nullptr;
    int rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp);
    if (rc) return rc;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, (int)n, st));
    h->launches++;
    return MKB_OK;
}

}  // namespace mkb

using namespace mkb;

// The fill kernel of a call, chosen once for the batch from its finest grid (the largest cutoff in voxels, cv):
//   runs     occ_fill_runs_kernel: 8 channels, no accumulate, 16-byte aligned output, cv <= 40 (voxelsize >= 0.125 A,
//            the range it is tested and measured on); the caller still drops it when the batch exceeds its index limits;
//   warp     otherwise, with <= 8 channels, occ_fill8v_kernel while a block's halo fits in V_ROWS cell rows (cv <= 14);
//   generic  otherwise occ_fill_kernel<CP>.
// MKB_OCC_V6 and MKB_OCC_GENERIC put the same input through a fallback, so tests can compare the kernels.
struct FillChoice {
    bool runs, warp;
};
static FillChoice choose_fill_kernel(int C, uint32_t flags, const float *out, const mkb_grid_desc *grids, int B) {
    int cv = 0;
    for (int b = 0; b < B; ++b) {
        if (!(grids[b].voxelsize > 0.0)) break;  // reported by the caller
        cv = std::max(cv, (int)std::ceil(CUTOFF_A / grids[b].voxelsize));
    }
    const bool generic = getenv("MKB_OCC_GENERIC") != nullptr;
    FillChoice f;
    f.runs = C == 8 && !(flags & MKB_OCC_ACCUMULATE) && (uintptr_t)out % 16 == 0 && cv <= 40 && !generic && !getenv("MKB_OCC_V6");
    f.warp = C <= 8 && ((1 + 2 * cv) / V_CELL + 1) * ((3 + 2 * cv) / V_CELL + 1) <= V_ROWS && !generic;
    return f;
}

static int occupancy_grid_batch_impl(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                                     const double *radii, const uint32_t *chanmask, int64_t n_atoms, int32_t C,
                                     const mkb_grid_desc *grids, int32_t B, float *out, uint32_t flags,
                                     uint32_t *blk_rank = nullptr, int64_t rank_capacity = 0, uint32_t *host_rank = nullptr) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (B < 0 || n_atoms < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (C < 1 || C > 32) return fail(h, MKB_ERR_BAD_ARG, "C=%d: 1..32 channels per call (split wider channel sets)", C);
    if (B == 0) return MKB_OK;
    if (!grids || !out) return fail(h, MKB_ERR_BAD_ARG, "null grids/out");
    if (n_atoms >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "n_atoms must be < 2^31");
    if (n_atoms > 0 && (!coords || (!sigmas && (!radii || !chanmask))))
        return fail(h, MKB_ERR_BAD_ARG, "null coords/sigmas");

    const FillChoice fill = choose_fill_kernel(C, flags, out, grids, B);
    const int cellsz = fill.warp ? V_CELL : TILE;

    std::vector<GridDev> gd((size_t)B);
    long long items = 0, tiles = 0, cells = 0, voxels = 0;
    for (int b = 0; b < B; ++b) {
        const mkb_grid_desc &s = grids[b];
        GridDev &g = gd[b];
        if (!(s.voxelsize > 0.0) || !std::isfinite(s.voxelsize))
            return fail(h, MKB_ERR_BAD_ARG, "grid %d: voxelsize must be positive and finite", b);
        if (s.atom_begin < 0 || s.atom_end < s.atom_begin || s.atom_end > n_atoms)
            return fail(h, MKB_ERR_BAD_ARG, "grid %d: bad atom range [%lld, %lld)", b, (long long)s.atom_begin,
                        (long long)s.atom_end);
        if (s.out_offset < 0) return fail(h, MKB_ERR_BAD_ARG, "grid %d: negative out_offset", b);
        const double cut = CUTOFF_A / s.voxelsize;
        if (cut > 4096.0) return fail(h, MKB_ERR_BAD_ARG, "grid %d: voxelsize %g too small", b, s.voxelsize);
        g.vs = s.voxelsize;
        g.inv_vs = 1.0 / s.voxelsize;
        g.cutv = (int)std::ceil(cut);
        g.rcells = (TILE - 1 + 2 * g.cutv) / TILE;
        if ((g.rcells + 1) * (g.rcells + 1) > MAX_ROWS)
            return fail(h, MKB_ERR_BAD_ARG, "grid %d: voxelsize %g too small for one call", b, s.voxelsize);
        g.cut2v = (float)(cut * cut);
        g.cut2v_lo = g.cut2v * (1.0f - GATE_BAND);
        g.cut2v_hi = g.cut2v * (1.0f + GATE_BAND);
        g.cell = cellsz;
        long long nt = 1, nc = 1;
        for (int d = 0; d < 3; ++d) {
            if (s.dims[d] <= 0) return fail(h, MKB_ERR_BAD_ARG, "grid %d: dims must be positive", b);
            if (!std::isfinite(s.origin[d])) return fail(h, MKB_ERR_BAD_ARG, "grid %d: origin not finite", b);
            g.origin[d] = s.origin[d];
            g.dims[d] = s.dims[d];
            g.tiles[d] = (s.dims[d] + TILE - 1) / TILE;
            g.cells[d] = (s.dims[d] + 2 * g.cutv + cellsz - 1) / cellsz;
            if (g.cells[d] > 1023) return fail(h, MKB_ERR_BAD_ARG, "grid %d: too many voxels along an axis for one call", b);
            nt *= g.tiles[d];
            nc *= g.cells[d];
        }
        g.atom_begin = s.atom_begin;
        g.atom_end = s.atom_end;
        g.out_offset = s.out_offset;
        g.item_base = items;
        g.tile_base = tiles;
        g.cell_base = cells;
        g.vox_base = voxels;
        g.blk_base = 0;
        voxels += (long long)s.dims[0] * s.dims[1] * s.dims[2];
        items += s.atom_end - s.atom_begin;
        tiles += nt;
        cells += nc;
    }
    if (tiles >= (1ll << 31) - 1) return fail(h, MKB_ERR_BAD_ARG, "too many tiles (%lld): split the batch", tiles);
    if (cells >= (1ll << 31) - 2 || items >= (1ll << 31))
        return fail(h, MKB_ERR_BAD_ARG, "batch too large (%lld cells, %lld atom items): split it", cells, items);

    // ---- default for 8 channels: per-tile candidate lists + persistent mask-run kernel with TMA stores (occ_runs.cuh)
    bool use_runs = fill.runs;
    std::vector<long long> ibase;
    long long run_blocks = 0, run_items = 0, ent_bound = 0;
    int list_table = 1;  // the list passes count per CTA in shared memory (occ_runs.cuh): off for fine voxels
    int run_zc = R_ZC;
    if (use_runs) {
        std::vector<long long> nblk((size_t)B), nitem((size_t)B), nent((size_t)B);
        // z blocks per queue item: 4 amortise the item set-up, but a small batch (strong scaling: 32 pockets per GPU) then
        // has ~2 items per warp and the heavy ones decide the tail -> finer items when there are few
        {
            long long it4 = 0;
            for (int b = 0; b < B; ++b)
                it4 += (long long)((gd[b].dims[0] + 3) / 4) * ((gd[b].dims[1] + 3) / 4) * (((gd[b].dims[2] + R_BZ - 1) / R_BZ + R_ZC - 1) / R_ZC);
            const long long warps = (long long)h->sm_count * MKB_R_MIN_CTAS * R_WARPS;
            run_zc = it4 >= 8 * warps ? R_ZC : (it4 >= 3 * warps ? 2 : 1);
        }
        for (int b = 0; b < B; ++b) {
            const GridDev &g = gd[b];
            const long long nbx = (g.dims[0] + 3) / 4, nby = (g.dims[1] + 3) / 4, nbz = (g.dims[2] + R_BZ - 1) / R_BZ;
            if (g.dims[0] + 2 * g.cutv + 2 >= 65536 || g.dims[1] + 2 * g.cutv + 2 >= 65536 || g.dims[2] + 2 * g.cutv + 2 >= 65536) use_runs = false;
            nblk[b] = nbx * nby * nbz;
            nitem[b] = nbx * nby * ((nbz + run_zc - 1) / run_zc);
            // tiles (8 x 8 x 8 voxels) one atom can reach: an interval of 2 reach voxels touches at most
            // floor((2 reach + 7) / 8) + 1 tiles; reach = the cutoff with the list walk's slack
            const double c2 = 2.0 * CUTOFF_A / g.vs * (1.0 + (double)R_LIST_SLACK);
            const long long rx = std::min<long long>(g.tiles[0], (long long)((c2 + 7) / 8) + 1),
                            ry = std::min<long long>(g.tiles[1], (long long)((c2 + 7) / 8) + 1),
                            rz = std::min<long long>(nbz, (long long)((c2 + R_BZ - 1) / R_BZ) + 1);
            nent[b] = (g.atom_end - g.atom_begin) * rx * ry * rz;
            if (rx * ry * rz > L_TABLE_MAX_REACH) list_table = 0;
            run_blocks += nblk[b]; run_items += nitem[b]; ent_bound += nent[b];
        }
        if (run_blocks >= (1ll << 31) - 64 || ent_bound >= (1ll << 32) - 1) use_runs = false;
        if (use_runs) {
            ibase.assign((size_t)B + 1, 0);
            long long bsum = 0;
            for (int b = 0; b < B; ++b) {
                gd[b].blk_base = bsum;
                bsum += nblk[b];
                ibase[b + 1] = ibase[b] + nitem[b];
            }
        }
    }
    if (blk_rank && !use_runs)
        return fail(h, MKB_ERR_UNSUPPORTED, "compact output needs the run kernel (8 channels, 16-byte aligned records, default kernel selection)");
    if (blk_rank && (flags & MKB_OCC_LAYOUT_CXYZ)) return fail(h, MKB_ERR_BAD_ARG, "compact output is voxel-major");
    if (blk_rank && rank_capacity < run_blocks + 1)
        return fail(h, MKB_ERR_BAD_ARG, "blk_rank holds %lld entries, the batch has %lld blocks + 1", (long long)rank_capacity, run_blocks);
    if (use_runs) {
        GridDev *d_grids;
        float4 *rec_pos;
        uint4 *rec_tag;
        unsigned *blk_count, *blk_start, *d_bitmap, *d_queue, *segs = nullptr, *seg_n = nullptr;
        uint2 *blk_ent;
        long long *d_ibase;
        unsigned long long *d_fix;
        int rc;
        const size_t ni = (size_t)std::max<long long>(items, 1);
        const long long n_words = cdiv(voxels, 32);
        const unsigned fix_cap = (unsigned)std::min<long long>(voxels, 1ll << 22);
        const size_t nslots = (size_t)tiles + 1;  // list slots (tile_base: 8x8x8 tiles) + 1: the total after the exclusive scan
        const long long list_ctas = cdiv(items, L_THREADS);
        if ((rc = scratch_get(h, S_DESC, (size_t)B, &d_grids))) return rc;
        if ((rc = scratch_get(h, S_SORT_PX, ni, &rec_pos))) return rc;
        if ((rc = scratch_get(h, S_SORT_PY, ni, &rec_tag))) return rc;
        // per tile: entries in the CTAs' table segments (blk_count), the direct insertions (blk_direct), the blocks with a
        // candidate (tile_bits); behind them the compact output's per-block flags
        if ((rc = scratch_get(h, S_CELL_COUNT, 3 * nslots + (blk_rank ? (size_t)run_blocks + 1 : 0), &blk_count))) return rc;
        unsigned *const blk_direct = blk_count + nslots, *const tile_bits = blk_direct + nslots, *const blk_flag = tile_bits + nslots;
        if (list_table && list_ctas > 0) {  // the count pass's table segments, read back by the fill pass
            if ((rc = scratch_get(h, S_BLK_SEGS, (size_t)list_ctas * (L_SEG_WORDS + 1), &segs))) return rc;
            seg_n = segs + (size_t)list_ctas * L_SEG_WORDS;
        }
        if ((rc = scratch_get(h, S_CELL_START, nslots, &blk_start))) return rc;
        if ((rc = scratch_get(h, S_BLK_ENT, (size_t)std::max<long long>(ent_bound, 1), &blk_ent))) return rc;
        if ((rc = scratch_get(h, S_BLOCK_BASE, (size_t)B + 1, &d_ibase))) return rc;
        if ((rc = scratch_get(h, S_BAND_BITMAP, (size_t)n_words, &d_bitmap))) return rc;
        if ((rc = scratch_get(h, S_QUEUE, (size_t)64, &d_queue))) return rc;
        if ((rc = scratch_get(h, S_FIX_LIST, (size_t)fix_cap + FIX_HDR, &d_fix))) return rc;
        // cub temp storage for the scans, sized before anything is enqueued
        unsigned *scan_tmp = nullptr;
        size_t scan_bytes = 0;
        const auto list_len = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), ListLength{blk_count, blk_direct});
        {
            size_t rank_bytes = 0;
            MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, list_len, blk_start, (int)nslots, st));
            MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, rank_bytes, blk_count, blk_start, (int)(run_blocks + 1), st));
            scan_bytes = std::max(scan_bytes, rank_bytes);
            void *tmp = nullptr;
            if ((rc = scratch_get(h, S_SCAN_TMP, scan_bytes, &tmp))) return rc;
            scan_tmp = static_cast<unsigned *>(tmp);
        }
        if (!h->aux_stream) {
            MKB_CUDA(h, cudaStreamCreateWithFlags(&h->aux_stream, cudaStreamNonBlocking));
            MKB_CUDA(h, cudaStreamCreateWithFlags(&h->aux_stream2, cudaStreamNonBlocking));
            for (auto &e : h->aux_ev) MKB_CUDA(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        }
        if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        {   // descriptors + item table: one upload from page-locked staging
            const size_t gbytes = sizeof(GridDev) * (size_t)B, ibytes = sizeof(long long) * ((size_t)B + 1);
            void *stage = nullptr;
            cudaEvent_t *sev = nullptr;
            if ((rc = host_stage_get(h, gbytes + ibytes, &stage, &sev))) return rc;
            memcpy(stage, gd.data(), gbytes);
            memcpy(static_cast<char *>(stage) + gbytes, ibase.data(), ibytes);
            MKB_CUDA(h, cudaMemcpyAsync(d_grids, stage, gbytes, cudaMemcpyHostToDevice, st));
            MKB_CUDA(h, cudaMemcpyAsync(d_ibase, static_cast<char *>(stage) + gbytes, ibytes, cudaMemcpyHostToDevice, st));
            MKB_CUDA(h, cudaEventRecord(*sev, st));
        }
        MKB_CUDA(h, cudaMemsetAsync(blk_count, 0, sizeof(unsigned) * 3 * nslots, st));
        MKB_CUDA(h, cudaMemsetAsync(d_bitmap, 0, sizeof(unsigned) * (size_t)n_words, st));
        MKB_CUDA(h, cudaMemsetAsync(d_queue, 0, sizeof(unsigned) * 64, st));
        MKB_CUDA(h, cudaMemsetAsync(d_fix, 0, sizeof(unsigned long long) * FIX_HDR, st));
        // the gate-band pre-pass (compute bound) runs beside the list build (atomic bound) on a side stream; small calls
        // keep it on the caller's stream (the fork / join costs more host time than the overlap saves)
        const bool band_aside = items >= 200000;
        if (items > 0) {
            cudaStream_t sb = band_aside ? h->aux_stream : st;
            if (band_aside) {
                MKB_CUDA(h, cudaEventRecord(h->aux_ev[0], st));
                MKB_CUDA(h, cudaStreamWaitEvent(sb, h->aux_ev[0], 0));
            }
            occ_band_kernel<<<(unsigned)cdiv(items, 128), 128, 0, sb>>>(coords, d_grids, B, items, d_bitmap, d_fix, fix_cap);
            MKB_LAUNCHED(h);
            if (band_aside) MKB_CUDA(h, cudaEventRecord(h->aux_ev[1], sb));
        }
        h->last_kernel = "occ_fill_runs_kernel";
        if (items > 0) {
            occ_prep_kernel<<<(unsigned)list_ctas, L_THREADS, 0, st>>>(coords, sigmas, radii, chanmask, d_grids, B, items, rec_pos, rec_tag,
                                                                       blk_count, blk_direct, tile_bits, segs, seg_n, list_table);
            MKB_LAUNCHED(h);
        }
        MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, list_len, blk_start, (int)nslots, st));
        h->launches++;
        if (items > 0) {
            occ_blk_fill_kernel<<<(unsigned)list_ctas, L_THREADS, 0, st>>>(d_grids, B, items, rec_pos, rec_tag, blk_direct, blk_start, segs, seg_n,
                                                                           blk_ent, list_table);
            MKB_LAUNCHED(h);
        }
        if (blk_rank) {  // record index of every non-empty block
            occ_blk_flag_kernel<<<(unsigned)cdiv(run_blocks + 1, 256), 256, 0, st>>>(d_grids, B, tile_bits, run_blocks, blk_flag);
            MKB_LAUNCHED(h);
            MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, blk_flag, blk_rank, (int)(run_blocks + 1), st));
            h->launches++;
            if (host_rank) {  // the block index leaves for the host NOW (side stream), before the fill kernel starts
                MKB_CUDA(h, cudaEventRecord(h->aux_ev[2], st));
                MKB_CUDA(h, cudaStreamWaitEvent(h->aux_stream2, h->aux_ev[2], 0));
                MKB_CUDA(h, cudaMemcpyAsync(host_rank, blk_rank, sizeof(uint32_t) * (size_t)(run_blocks + 1), cudaMemcpyDeviceToHost, h->aux_stream2));
                MKB_CUDA(h, cudaEventRecord(h->aux_ev[3], h->aux_stream2));
                h->index_pending = true;
            }
        }
        {
            RunParams rp;
            rp.grids = d_grids; rp.B = B;
            rp.rec_pos = rec_pos; rp.rec_tag = rec_tag; rp.blk_start = blk_start; rp.tile_bits = tile_bits; rp.blk_ent = blk_ent;
            rp.sigmas = sigmas; rp.out = out;
            rp.item_base = d_ibase; rp.queue = d_queue;
            rp.total_items = (unsigned)run_items;
            rp.cmajor = (flags & MKB_OCC_LAYOUT_CXYZ) ? 1 : 0;
            rp.blk_rank = blk_rank;
            rp.sparse_dense = host_rank ? 1 : 0;
            bool uni = true;
            const GridDev &g0d = gd[0];
            const long long nvox0 = (long long)g0d.dims[0] * g0d.dims[1] * g0d.dims[2];
            for (int b = 0; b < B && uni; ++b) {
                const GridDev &g = gd[b];
                uni = g.dims[0] == g0d.dims[0] && g.dims[1] == g0d.dims[1] && g.dims[2] == g0d.dims[2] && g.vs == g0d.vs &&
                      g.out_offset == g0d.out_offset + b * nvox0;
            }
            rp.u = g0d;
            rp.u_out_stride = nvox0;
            rp.u_ipg = (unsigned)(ibase[1] - ibase[0]);
            rp.u_nby = (unsigned)((g0d.dims[1] + 3) / 4);
            rp.u_nzc = (unsigned)(((g0d.dims[2] + R_BZ - 1) / R_BZ + run_zc - 1) / run_zc);
            rp.zc = run_zc;
            rp.u_bpg = (unsigned)(B > 1 ? gd[1].blk_base - g0d.blk_base : 0);
            rp.u_tpg = (unsigned)(B > 1 ? gd[1].tile_base - g0d.tile_base : 0);
            if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
            const unsigned nctas = (unsigned)std::min<long long>((long long)h->sm_count * MKB_R_MIN_CTAS, cdiv((long long)rp.total_items, R_WARPS));
            rp.use_tmap = 0;
            CUtensorMap tmap;
            memset(&tmap, 0, sizeof(tmap));
            // dense uniform output in device memory (the to-host route writes mapped host memory: row copies)
            if (uni && !rp.cmajor && !rp.blk_rank && !getenv("MKB_OCC_NO_TMAP"))
                rp.use_tmap = occ_make_tmap(&tmap, out + g0d.out_offset * 8, g0d.dims[0], g0d.dims[1], g0d.dims[2], B, nvox0) ? 1 : 0;
            if (nctas > 0) {
                if (uni) occ_fill_runs_kernel<true><<<nctas, R_WARPS * 32, 0, st>>>(rp, tmap);
                else occ_fill_runs_kernel<false><<<nctas, R_WARPS * 32, 0, st>>>(rp, tmap);
                MKB_LAUNCHED(h);
            }
        }
        if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
        if (items > 0) {
            if (band_aside) MKB_CUDA(h, cudaStreamWaitEvent(st, h->aux_ev[1], 0));
            const unsigned fg = (unsigned)h->sm_count * 4;
            const int cm = (flags & MKB_OCC_LAYOUT_CXYZ) ? 1 : 0;
            const uint32_t *fix_rank = host_rank ? nullptr : blk_rank;  // dense addressing in the to-host mode
            occ_fix_list_kernel<<<fg, 256, 0, st>>>(d_grids, B, d_fix, fix_cap, coords, sigmas, radii, chanmask, rec_tag, blk_start, blk_ent, out, cm, fix_rank);
            MKB_LAUNCHED(h);
            occ_fix_scan_kernel<<<fg, 256, 0, st>>>(d_grids, B, n_words, d_bitmap, d_fix, fix_cap, coords, sigmas, radii, chanmask,
                                                    rec_tag, blk_start, blk_ent, out, cm, fix_rank);
            MKB_LAUNCHED(h);
        }
        return MKB_OK;
    }
    (void)ent_bound;

    GridDev *d_grids;
    int *item_cell;
    unsigned *item_slot, *cell_count, *cell_start;
    float4 *rec_pos;
    uint4 *rec_tag;
    int rc;
    const size_t ni = (size_t)std::max<long long>(items, 1);
    if ((rc = scratch_get(h, S_DESC, (size_t)B, &d_grids))) return rc;
    if ((rc = scratch_get(h, S_ITEM_CELL, ni, &item_cell))) return rc;
    if ((rc = scratch_get(h, S_ITEM_SLOT, ni, &item_slot))) return rc;
    if ((rc = scratch_get(h, S_CELL_COUNT, (size_t)cells + 1, &cell_count))) return rc;
    if ((rc = scratch_get(h, S_CELL_START, (size_t)cells + 1, &cell_start))) return rc;
    if ((rc = scratch_get(h, S_SORT_PX, ni, &rec_pos))) return rc;
    if ((rc = scratch_get(h, S_SORT_PY, ni, &rec_tag))) return rc;

    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_grids, gd.data(), sizeof(GridDev) * (size_t)B, cudaMemcpyHostToDevice, st));
    MKB_CUDA(h, cudaMemsetAsync(cell_count, 0, sizeof(unsigned) * ((size_t)cells + 1), st));
    if (items > 0) {
        const int nb = (int)cdiv(items, 256);
        occ_bin_kernel<<<nb, 256, 0, st>>>(coords, d_grids, B, items, item_cell, item_slot, cell_count);
        MKB_LAUNCHED(h);
    }
    if ((rc = scan_u32(h, st, cell_count, cell_start, cells + 1))) return rc;
    if (items > 0) {
        const int nb = (int)cdiv(items, 256);
        occ_scatter_kernel<<<nb, 256, 0, st>>>(coords, sigmas, radii, chanmask, C, d_grids, B, items, item_cell, item_slot,
                                               cell_start, rec_pos, rec_tag);
        MKB_LAUNCHED(h);
    }
    FillParams fp;
    fp.grids = d_grids; fp.B = B; fp.C = C;
    fp.rec_pos = rec_pos; fp.rec_tag = rec_tag;
    fp.cell_start = cell_start; fp.coords = coords; fp.sigmas = sigmas; fp.out = out; fp.flags = flags;
    fp.cmajor = (flags & MKB_OCC_LAYOUT_CXYZ) ? 1 : 0;
    fp.vec_ok = (C == 8 && ((uintptr_t)out % 16 == 0) && !fp.cmajor) ? 1 : 0;
    fp.txp_shift = 0;

    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    if (fill.warp) {
        // per-block halo counts (thread per block), then the warp-per-block kernel on 2x4x8-voxel blocks:
        // grid = (z-blocks, y-blocks, grid << sh | x-block)
        std::vector<long long> bbase((size_t)B + 1, 0);
        long long maxblk = 0;
        for (int b = 0; b < B; ++b) {
            const long long nbk = (long long)((gd[b].dims[0] + 1) / 2) * ((gd[b].dims[1] + 3) / 4) * ((gd[b].dims[2] + V_BZ - 1) / V_BZ);
            bbase[b + 1] = bbase[b] + nbk;
            maxblk = std::max(maxblk, nbk);
        }
        long long *d_bbase;
        unsigned *d_btotal;
        if ((rc = scratch_get(h, S_BLOCK_BASE, (size_t)B + 1, &d_bbase))) return rc;
        if ((rc = scratch_get(h, S_TILE_TOTAL, (size_t)bbase[B], &d_btotal))) return rc;
        MKB_CUDA(h, cudaMemcpyAsync(d_bbase, bbase.data(), sizeof(long long) * ((size_t)B + 1), cudaMemcpyHostToDevice, st));
        for (int c0 = 0; c0 < B; c0 += 65535) {
            const int cn = std::min(65535, B - c0);
            occ_block_total_v_kernel<<<dim3((unsigned)cdiv(maxblk, 256), (unsigned)cn), 256, 0, st>>>(d_grids + c0, cell_start, d_bbase + c0, d_btotal);
            MKB_LAUNCHED(h);
        }
        int b0 = 0;
        while (b0 < B) {
            int mx = 1, my = 1, mz = 1, sh = 0, nb = 0;
            for (int b = b0; b < B; ++b) {  // extend the chunk while gridDim.z stays legal
                const int ax = std::max(mx, (gd[b].dims[0] + 1) / 2);
                int s2 = 0;
                while ((1 << s2) < ax) ++s2;
                if (((long long)(nb + 1) << s2) > 65535) break;
                mx = ax; sh = s2; ++nb;
                my = std::max(my, (gd[b].dims[1] + 3) / 4);
                mz = std::max(mz, (gd[b].dims[2] + V_BZ - 1) / V_BZ);
            }
            if (nb == 0 || my > 65535) return fail(h, MKB_ERR_BAD_ARG, "grid %d too large for one launch", b0);
            FillParams fq = fp;
            fq.grids = d_grids + b0;
            fq.B = nb;
            fq.txp_shift = sh;
            // uniform chunk: same shape everywhere and regularly spaced output / cells / blocks
            bool uni = true;
            const GridDev &g0 = gd[b0];
            const long long nvox0 = (long long)g0.dims[0] * g0.dims[1] * g0.dims[2];
            const long long ncell0 = (long long)g0.cells[0] * g0.cells[1] * g0.cells[2];
            for (int b = b0; b < b0 + nb && uni; ++b) {
                const GridDev &g = gd[b];
                uni = g.dims[0] == g0.dims[0] && g.dims[1] == g0.dims[1] && g.dims[2] == g0.dims[2] && g.vs == g0.vs &&
                      g.out_offset == g0.out_offset + (b - b0) * nvox0 && g.cell_base == g0.cell_base + (b - b0) * ncell0;
            }
            fq.u = g0;
            fq.u_out_stride = nvox0;
            fq.u_cell_stride = ncell0;
            fq.u_block_base = bbase[b0];
            fq.u_block_stride = bbase[b0 + 1] - bbase[b0];
            {
                const float band = g0.cut2v_hi - g0.cut2v_lo;
                memcpy(&fq.u_band_bits, &band, sizeof(float));
            }
            h->last_kernel = "occ_fill8v_kernel";
            const dim3 vgrid((unsigned)cdiv(mz, V_WARPS), (unsigned)my, (unsigned)(nb << sh));
            if (uni) occ_fill8v_kernel<true><<<vgrid, V_WARPS * 32, 0, st>>>(fq, d_bbase + b0, d_btotal);
            else occ_fill8v_kernel<false><<<vgrid, V_WARPS * 32, 0, st>>>(fq, d_bbase + b0, d_btotal);
            MKB_LAUNCHED(h);
            b0 += nb;
        }
    }
    for (int b0 = 0; b0 < B && !fill.warp; b0 += 65535) {  // tile kernel: blockIdx.y = grid of the batch
        const int nb = std::min(65535, B - b0);
        fp.grids = d_grids + b0;
        fp.B = nb;
        long long mt = 0;
        for (int b = b0; b < b0 + nb; ++b) mt = std::max<long long>(mt, (long long)gd[b].tiles[0] * gd[b].tiles[1] * gd[b].tiles[2]);
        const dim3 grid((unsigned)mt, (unsigned)nb);
        h->last_kernel = "occ_fill_kernel";
        if (C <= 8) occ_fill_kernel<8><<<grid, FILL_THREADS, 0, st>>>(fp);
        else if (C <= 16) occ_fill_kernel<16><<<grid, FILL_THREADS, 0, st>>>(fp);
        else occ_fill_kernel<32><<<grid, FILL_THREADS, 0, st>>>(fp);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_occupancy_grid_batch(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                                        int64_t n_atoms, int32_t C, const mkb_grid_desc *grids, int32_t B,
                                        float *out, uint32_t flags) {
    if (h && n_atoms > 0 && !sigmas) return fail(h, MKB_ERR_BAD_ARG, "null coords/sigmas");
    return occupancy_grid_batch_impl(h, stream, coords, sigmas, nullptr, nullptr, n_atoms, C, grids, B, out, flags);
}

extern "C" int mkb_occupancy_grid_batch_masked(mkb_handle_t h, void *stream, const float *coords, const double *radii,
                                               const uint32_t *chanmask, int64_t n_atoms, int32_t C,
                                               const mkb_grid_desc *grids, int32_t B, float *out, uint32_t flags) {
    if (h && n_atoms > 0 && (!radii || !chanmask)) return fail(h, MKB_ERR_BAD_ARG, "null radii/chanmask");
    return occupancy_grid_batch_impl(h, stream, coords, nullptr, radii, chanmask, n_atoms, C, grids, B, out, flags);
}

extern "C" int mkb_occupancy_grid_batch_compact(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                                                const double *radii, const uint32_t *chanmask, int64_t n_atoms,
                                                const mkb_grid_desc *grids, int32_t B, float *records, uint32_t *blk_rank,
                                                int64_t rank_capacity) {
    if (h && n_atoms > 0 && !sigmas && (!radii || !chanmask)) return fail(h, MKB_ERR_BAD_ARG, "null sigmas and radii/chanmask");
    if (h && !blk_rank) return fail(h, MKB_ERR_BAD_ARG, "null blk_rank");
    return occupancy_grid_batch_impl(h, stream, coords, sigmas, sigmas ? nullptr : radii, sigmas ? nullptr : chanmask, n_atoms, 8, grids,
                                     B, records, 0u, blk_rank, rank_capacity);
}

extern "C" int mkb_occupancy_grid_batch_to_host(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                                                const double *radii, const uint32_t *chanmask, int64_t n_atoms,
                                                const mkb_grid_desc *grids, int32_t B, float *out_mapped, uint32_t *blk_rank,
                                                int64_t rank_capacity, uint32_t *host_rank) {
    if (h && n_atoms > 0 && !sigmas && (!radii || !chanmask)) return fail(h, MKB_ERR_BAD_ARG, "null sigmas and radii/chanmask");
    if (h && (!blk_rank || !host_rank)) return fail(h, MKB_ERR_BAD_ARG, "null blk_rank / host_rank");
    return occupancy_grid_batch_impl(h, stream, coords, sigmas, sigmas ? nullptr : radii, sigmas ? nullptr : chanmask, n_atoms, 8, grids,
                                     B, out_mapped, 0u, blk_rank, rank_capacity, host_rank);
}

extern "C" int mkb_occupancy_wait_index(mkb_handle_t h) {
    MKB_ENTER(h);
    if (h->index_pending) {
        MKB_CUDA(h, cudaEventSynchronize(h->aux_ev[3]));
        h->index_pending = false;
    }
    return MKB_OK;
}

extern "C" int64_t mkb_occupancy_compact_blocks(const mkb_grid_desc *grids, int32_t B) {
    int64_t n = 0;
    for (int b = 0; b < B; ++b)
        n += (int64_t)((grids[b].dims[0] + 3) / 4) * ((grids[b].dims[1] + 3) / 4) * ((grids[b].dims[2] + R_BZ - 1) / R_BZ);
    return n;
}

// Host side of the compact transfer: grids [g0, g1) are rebuilt in the caller's dense (voxel-major, 8 channel) array from
// the 4 KB block records; blocks without a record are zero-filled.  `blk_rank` is the whole batch's table (host copy),
// `records` points at record `rec0` (the first record of grid g0: a chunk of grids is a contiguous range of records).
// The expansion writes every byte of the dense array exactly once and never reads it back: non-temporal stores skip the
// read-for-ownership of ordinary stores (half the memory traffic).  Rows start on 32-byte (voxel) boundaries.
#if defined(__SSE2__) || defined(__x86_64__)
#include <emmintrin.h>
static inline void stream_zero(float *d, int n) {
    const __m128i z = _mm_setzero_si128();
    for (int i = 0; i < n; i += 4) _mm_stream_si128(reinterpret_cast<__m128i *>(d + i), z);
}
static inline void stream_zero(double *d, int n) {
    const __m128i z = _mm_setzero_si128();
    for (int i = 0; i < n; i += 2) _mm_stream_si128(reinterpret_cast<__m128i *>(d + i), z);
}
static inline void stream_copy(float *d, const float *s, int n) {
    for (int i = 0; i < n; i += 4) _mm_stream_si128(reinterpret_cast<__m128i *>(d + i), _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + i)));
}
static inline void stream_copy(double *d, const float *s, int n) {
    for (int i = 0; i < n; i += 4) {
        const __m128 v = _mm_loadu_ps(s + i);
        _mm_stream_pd(d + i, _mm_cvtps_pd(v));
        _mm_stream_pd(d + i + 2, _mm_cvtps_pd(_mm_movehl_ps(v, v)));
    }
}
static inline void stream_fence() { _mm_sfence(); }
#else
static inline void stream_zero(float *d, int n) { memset(d, 0, (size_t)n * 4); }
static inline void stream_zero(double *d, int n) { memset(d, 0, (size_t)n * 8); }
static inline void stream_copy(float *d, const float *s, int n) { memcpy(d, s, (size_t)n * 4); }
static inline void stream_copy(double *d, const float *s, int n) { for (int i = 0; i < n; ++i) d[i] = (double)s[i]; }
static inline void stream_fence() {}
#endif

template <typename T>
static int expand_host_impl(const mkb_grid_desc *grids, int32_t g0, int32_t g1, const uint32_t *blk_rank, const float *records,
                            int64_t rec0, T *out, int32_t n_threads) {
    std::vector<int64_t> bbase((size_t)g1 + 1, 0);
    for (int b = 0; b < g1; ++b)
        bbase[b + 1] = bbase[b] + (int64_t)((grids[b].dims[0] + 3) / 4) * ((grids[b].dims[1] + 3) / 4) * ((grids[b].dims[2] + R_BZ - 1) / R_BZ);
    // work items: (grid, x block row); threads take them round robin
    std::vector<std::pair<int, int>> items;
    for (int b = g0; b < g1; ++b)
        for (int bx = 0; bx < (grids[b].dims[0] + 3) / 4; ++bx) items.emplace_back(b, bx);
    const int nt = std::max(1, std::min<int>(n_threads, (int)items.size()));
    auto work = [&](int t) {
        for (size_t i = (size_t)t; i < items.size(); i += (size_t)nt) {
            const int b = items[i].first, bx = items[i].second;
            const mkb_grid_desc &g = grids[b];
            const int nx = g.dims[0], ny = g.dims[1], nz = g.dims[2];
            const int nby = (ny + 3) / 4, nbz = (nz + R_BZ - 1) / R_BZ;
            T *const gout = out + g.out_offset * 8;
            for (int by = 0; by < nby; ++by)
                for (int k = 0; k < 4 && bx * 4 + k < nx; ++k)
                    for (int l = 0; l < 4 && by * 4 + l < ny; ++l) {
                        T *row = gout + ((int64_t)(bx * 4 + k) * ny + (by * 4 + l)) * nz * 8;
                        const int64_t bid0 = bbase[b] + ((int64_t)bx * nby + by) * nbz;
                        for (int bz = 0; bz < nbz; ++bz) {
                            const int nfl = std::min(R_BZ, nz - bz * R_BZ) * 8;
                            const uint32_t r = blk_rank[bid0 + bz];
                            if (blk_rank[bid0 + bz + 1] != r) {
                                if (records) stream_copy(row + bz * 64, records + ((int64_t)r - rec0) * 1024 + (k * 4 + l) * 64, nfl);
                            } else stream_zero(row + bz * 64, nfl);
                        }
                    }
        }
        stream_fence();
    };
    if (nt == 1) { work(0); return MKB_OK; }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back(work, t);
    for (auto &x : th) x.join();
    return MKB_OK;
}

// Host side of the compact transfer: grids [g0, g1) are rebuilt in the caller's dense (voxel-major, 8 channel) array from
// the 4 KB block records; blocks without a record are zero-filled.  `blk_rank` is the whole batch's table (host copy),
// `records` points at record `rec0` (the first record of grid g0: a chunk of grids is a contiguous range of records).
// out_f64 != 0: `out` is float64 (the reference's dtype, voxeldescriptors.py:531) and the upcast happens here, threaded.
extern "C" int mkb_occupancy_expand_host(const mkb_grid_desc *grids, int32_t g0, int32_t g1, const uint32_t *blk_rank,
                                         const float *records, int64_t rec0, void *out, int32_t out_f64, int32_t n_threads) {
    if (!grids || !blk_rank || !out || g0 < 0 || g1 < g0) return MKB_ERR_BAD_ARG;
    if (out_f64) return expand_host_impl<double>(grids, g0, g1, blk_rank, records, rec0, static_cast<double *>(out), n_threads);
    return expand_host_impl<float>(grids, g0, g1, blk_rank, records, rec0, static_cast<float *>(out), n_threads);
}

extern "C" int mkb_occupancy_points(mkb_handle_t h, void *stream, const double *centers, int64_t M,
                                    const float *coords, const double *sigmas, int64_t n_atoms, int32_t C,
                                    float *out, uint32_t flags) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (M < 0 || n_atoms < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (C < 1 || C > 32) return fail(h, MKB_ERR_BAD_ARG, "C=%d: 1..32 channels per call", C);
    if (M == 0) return MKB_OK;
    if (!centers || !out) return fail(h, MKB_ERR_BAD_ARG, "null centers/out");
    if (n_atoms >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "n_atoms must be < 2^31");
    if (n_atoms > 0 && (!coords || !sigmas)) return fail(h, MKB_ERR_BAD_ARG, "null coords/sigmas");

    unsigned nb = 1024;
    while ((long long)nb < 2 * n_atoms && nb < (1u << 22)) nb <<= 1;
    const unsigned hmask = nb - 1;
    int *item_bucket;
    unsigned *item_slot, *bcount, *bstart, *order;
    float *s2;
    int rc;
    const size_t na = (size_t)std::max<long long>(n_atoms, 1);
    if ((rc = scratch_get(h, S_ITEM_CELL, na, &item_bucket))) return rc;
    if ((rc = scratch_get(h, S_ITEM_SLOT, na, &item_slot))) return rc;
    if ((rc = scratch_get(h, S_CELL_COUNT, (size_t)nb + 1, &bcount))) return rc;
    if ((rc = scratch_get(h, S_PT_BUCKET, (size_t)nb + 1, &bstart))) return rc;
    if ((rc = scratch_get(h, S_PT_ORDER, na, &order))) return rc;
    if ((rc = scratch_get(h, S_PT_S2, na * (size_t)C, &s2))) return rc;
    MKB_CUDA(h, cudaMemsetAsync(bcount, 0, sizeof(unsigned) * ((size_t)nb + 1), st));
    if (n_atoms > 0) {
        const int g1 = (int)cdiv(n_atoms, 256);
        pt_bin_kernel<<<g1, 256, 0, st>>>(coords, n_atoms, hmask, item_bucket, item_slot, bcount);
        MKB_LAUNCHED(h);
        pt_sigma_kernel<<<(int)cdiv(n_atoms * C, 256), 256, 0, st>>>(sigmas, n_atoms * C, s2);
        MKB_LAUNCHED(h);
    }
    if ((rc = scan_u32(h, st, bcount, bstart, (long long)nb + 1))) return rc;
    if (n_atoms > 0) {
        pt_order_kernel<<<(int)cdiv(n_atoms, 256), 256, 0, st>>>(n_atoms, item_bucket, item_slot, bstart, order);
        MKB_LAUNCHED(h);
    }
    const unsigned g2 = (unsigned)cdiv(M, 128);
    if (C <= 8) occ_points_kernel<8><<<g2, 128, 0, st>>>(centers, M, coords, s2, sigmas, C, hmask, bstart, order, out, flags);
    else if (C <= 16) occ_points_kernel<16><<<g2, 128, 0, st>>>(centers, M, coords, s2, sigmas, C, hmask, bstart, order, out, flags);
    else occ_points_kernel<32><<<g2, 128, 0, st>>>(centers, M, coords, s2, sigmas, C, hmask, bstart, order, out, flags);
    MKB_LAUNCHED(h);
    return MKB_OK;
}
