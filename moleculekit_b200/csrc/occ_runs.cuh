// occ_runs.cuh -- K1, the default 8-channel occupancy fill (v10): per-block candidate lists + a persistent "mask-run" kernel.
// Included by occupancy.cu (after GridDev / occ_value).  Replaces the inner loop of
// moleculekit/occupancy_utils/occupancy_utils.pyx:46-61.  DESIGN.md section 3 has the derivations; the superseded variants
// (float-compare gate with predicated FMNMX, scalar FFMA hot loop, row-copy stores, in-register record gathers, jump-table
// flush, FFMA.SAT gate ...) are in the git history of this file together with their compile-time selectors.
//
//   * K2' (occ_prep_kernel / occ_blk_fill_kernel): every atom is appended to the candidate list of each 4x4x8-voxel
//     block it can reach (~16 blocks per atom at 1 A) -- count, scan, fill.  The fill kernel reads its list; no block
//     scans cell rows.
//   * value = max_a [d2 < cut2] f(sigma^2 / d2) with f monotone: the kernel tracks  r = d2 / sigma^2  as a MIN and applies f
//     once per voxel-channel; no reciprocal per pair.
//   * One warp owns a block; a lane owns the 4 voxels of one x-row (they share dy, dz).  The candidate is WARP-UNIFORM (two
//     LDS.128 broadcasts), so its channel mask is uniform too: candidates are counting-sorted by mask into runs (lane-parallel,
//     shared-memory histogram), a run keeps ONE scalar running minimum per voxel, and the channel update happens once per
//     run (low mask nibble) or once per group of runs that share the high nibble -- not once per pair.
//   * The 5 A gate is the float OVERFLOW of d2: the records carry differences scaled by lambda = 2^64 / cut, so
//     U = dx^2 + dy^2 + dz^2 = d2 2^128 / cut2 rounds to +inf exactly when the pair is outside the gate (threshold good to 3e-8;
//     tests/test_gate_scheme_cpu.py restates the arithmetic).  r = U w with w = 1 / (sigma lambda)^2 (inf stays inf) and the
//     minimum is an unpredicated FMNMX -- no compare, no predicate.  w is a denormal for sigma > 2.5 A
//     (cut2 / sigma^2 < 4): FMUL handles denormals at full rate; w then keeps 21 + log2(cut2 / sigma^2) bits.
//   * Per candidate a lane evaluates (dy, dz), their squares and sum once, then U and r of its four voxels: 13 FMA-pipe
//     instructions; the products and the sum are rounded on their own (no contraction), so r does not depend on the compiler.
//   * Pairs whose d2 lies within 2e-6 (relative) of the gate -- where float32 could decide differently from the reference's
//     float64 -- are found by a per-atom pre-pass (occ_band_kernel: the two lattice crossings of every (y, z) row of the
//     cutoff sphere) and their voxels are recomputed in float64 with the reference's operation order by occ_fix_*_kernel.
//   * Persistent CTAs (5 per SM x 4 warps, 96 registers) pull (x, y, 4 z-blocks) items from an atomic queue.  The record pass
//     gathers the per-atom data with cp.async straight into the candidates' sorted slots.  Results are staged in shared
//     memory in the output layout; a block of a dense uniform batch leaves as ONE TMA tensor store (cp.async.bulk.tensor.4d,
//     SASS UTMASTG; 4-D tensor map built per call), other outputs as cp.async.bulk row copies (UBLKCP); blocks without any
//     atom in reach (~65 %) are copies from a zeroed shared-memory tile, no math.
//   Tried and dropped: a queue that runs two items ahead (the second decode costs more issue slots than the latency it
//   hides); peeling the first candidate of a run; requesting the next z block's list words during the epilogue (the extra
//   live registers spill); 7 CTAs x 72 registers; 160 / 192 candidates per round; 2 z blocks per item.
#pragma once

namespace mkb {

constexpr int R_BZ = 8;          // block = 4 x 4 x 8 voxels
#ifndef MKB_R_CAP
#define MKB_R_CAP 224
#endif
constexpr int R_CAP = MKB_R_CAP;  // candidates per round (the 4 KB output stage aliases the records)
#ifndef MKB_R_WARPS
#define MKB_R_WARPS 4
#endif
constexpr int R_WARPS = MKB_R_WARPS;
#ifndef MKB_R_MIN_CTAS
#define MKB_R_MIN_CTAS 5         // 5 x 4 warps with 96 registers: at 6 x 80 the sm_90a build spills (4 % slower on an H100 SXM, 700 W)
#endif
#ifndef MKB_R_ZC
#define MKB_R_ZC 4               // consecutive z blocks per queue item
#endif
constexpr int R_ZC = MKB_R_ZC;
// per warp and candidate: x differences 16 | (-y, -z, w, tag) 16 | mask 1 | rank 1 bytes, then the 512-byte histogram
constexpr int R_WARP_BYTES = ((R_CAP * 34 + 512 + 127) / 128) * 128;
static_assert(R_CAP % 32 == 0 && R_CAP * 32 >= 4096 && R_WARP_BYTES % 128 == 0, "bad R_CAP");
constexpr float R_GATE_HUGE = 8.507059173023462e37f;  // 2^126: the epilogue's "no atom reached this voxel-channel" bound
constexpr float R_LIST_SLACK = 2e-4f;                 // relative slack of the block lists' reach test (float32 positions)

struct RunParams {
    const GridDev *grids;
    int B;
    const float4 *rec_pos;       // per atom item: position minus its nearest lattice point (voxel units), -
    const uint4 *rec_tag;        // mask | multi << 8 | lattice z << 16, atom row, lattice x | y << 16, 1/sigma
    const unsigned *blk_start;   // [blocks + 1] exclusive offsets of the per-block candidate lists
    const uint2 *blk_ent;        // (atom item, mask | multi << 8)
    const double *sigmas;        // multi-sigma atoms only
    float *out;
    const long long *item_base;  // [B + 1]: first queue item of every grid (item = 4 x 4 voxels in x, y and R_ZC blocks in z)
    unsigned item0;              // first item of this launch's chunk of grids (queue ids are chunk-local)
    int zc;                      // z blocks per item: R_ZC, or fewer when the batch has too few items to balance the resident warps
    unsigned *queue;
    unsigned total_items;
    int cmajor;                  // MKB_OCC_LAYOUT_CXYZ: grid stored [C][nx][ny][nz]; plain 32-byte-segment stores instead of TMA rows
    const unsigned *blk_rank;    // compact output (mkb_occupancy_grid_batch_compact): exclusive count of non-empty blocks; block
                                 // b with atoms in reach is one 4 KB record [4 x][4 y][8 z][8 ch] at out + 1024 * blk_rank[b],
                                 // empty blocks are not written at all; nullptr = the dense grid
    int use_tmap;                // the kernel's tensor-map argument describes `out` (dense, uniform, device memory)
    int sparse_dense;            // with blk_rank: keep the DENSE addressing (out may be mapped host memory) and only skip the empty
                                 // blocks -- the host zero-fills them meanwhile (mkb_occupancy_grid_batch_to_host)
    // uniform batches: descriptor of the first grid + strides (constant-bank operands)
    GridDev u;
    long long u_out_stride;
    unsigned u_ipg, u_nby, u_nzc, u_bpg;  // items per grid, y blocks, z chunks, blocks per grid
};

// ---------------------------------------------------------------------------------------------------------
// K2': records in atom order + per-block candidate lists.
// ---------------------------------------------------------------------------------------------------------
// blocks (4 x 4 x 8 voxels, voxel centres at integers) within `reach` of the point p; f(block id inside the grid)
template <class F>
__device__ __forceinline__ void for_each_block_in_reach(const GridDev &g, float px, float py, float pz, F f) {
    const int nbx = (g.dims[0] + 3) >> 2, nby = (g.dims[1] + 3) >> 2, nbz = (g.dims[2] + R_BZ - 1) / R_BZ;
    const float reach2 = g.cut2v * (1.0f + R_LIST_SLACK);
    const float reach = sqrtf(reach2) * (1.0f + 1e-6f);
    const int bx0 = max(0, (int)ceilf((px - reach - 3.0f) * 0.25f)), bx1 = min(nbx - 1, (int)floorf((px + reach) * 0.25f));
    const int by0 = max(0, (int)ceilf((py - reach - 3.0f) * 0.25f)), by1 = min(nby - 1, (int)floorf((py + reach) * 0.25f));
    const int bz0 = max(0, (int)ceilf((pz - reach - 7.0f) * 0.125f)), bz1 = min(nbz - 1, (int)floorf((pz + reach) * 0.125f));
    for (int bx = bx0; bx <= bx1; ++bx) {
        const float dx = fmaxf(fmaxf((float)(4 * bx) - px, px - (float)(4 * bx + 3)), 0.0f);
        for (int by = by0; by <= by1; ++by) {
            const float dy = fmaxf(fmaxf((float)(4 * by) - py, py - (float)(4 * by + 3)), 0.0f);
            const float dxy = fmaf(dy, dy, dx * dx);
            if (dxy > reach2) continue;
            for (int bz = bz0; bz <= bz1; ++bz) {
                const float dz = fmaxf(fmaxf((float)(R_BZ * bz) - pz, pz - (float)(R_BZ * bz + R_BZ - 1)), 0.0f);
                if (fmaf(dz, dz, dxy) <= reach2) f((bx * nby + by) * nbz + bz);
            }
        }
    }
}

// per atom item: record + block counts.  sigma handling as occ_scatter_kernel (one sigma + channel mask; several
// distinct sigmas -> multi flag and the per-channel path of the fill kernel).
__global__ void __launch_bounds__(128) occ_prep_kernel(const float *__restrict__ coords, const double *__restrict__ sigmas,
                                                       const double *__restrict__ radii, const unsigned *__restrict__ chanmask,
                                                       const GridDev *__restrict__ grids, int B, long long it0, long long n_items,
                                                       float4 *__restrict__ rec_pos, uint4 *__restrict__ rec_tag,
                                                       unsigned *__restrict__ blk_count) {
    const long long it = it0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (it >= it0 + n_items) return;
    const int b = find_grid_item(grids, B, it);
    const GridDev &g = grids[b];
    const long long a = g.atom_begin + (it - g.item_base);
    int ip[3];
    float f[3];
    bool live = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double pv = ((double)coords[3 * a + d] - g.origin[d]) * g.inv_vs;
        // atoms farther than the 5 A halo from the grid cannot touch any voxel (NaN fails both tests)
        live = live && (pv >= -(double)g.cutv - 0.5) && (pv <= (double)(g.dims[d] - 1 + g.cutv) + 0.5);
        const double r = live ? rint(pv) : 0.0;
        ip[d] = (int)r;
        f[d] = (float)(pv - r);  // |f| <= 0.5: absolute error <= 3e-8 voxel
    }
    double first = 0.0;
    unsigned m = 0;
    bool multi = false;
    if (sigmas) {
        const double *sg = sigmas + a * 8;
        for (int h = 0; h < 8; ++h) {
            const double s = sg[h];
            if (s == 0.0 || s != s) continue;  // sigma == 0 skipped (pyx:56); NaN never wins the max (pyx:61)
            if (m == 0) { first = s; m = 1u << h; }
            else if (s == first) m |= 1u << h;
            else multi = true;
        }
    } else {
        const double r = radii[a];
        const unsigned mm = chanmask[a] & 0xffu;
        if (mm && !(r == 0.0 || r != r)) { first = r; m = mm; }
    }
    live = live && m != 0;
    const double sv = first * g.inv_vs;  // sigma in voxel units
    const float sw = m ? (float)(1.0 / fabs(sv)) : 0.0f;
    const int off = g.cutv + 1;
    rec_pos[it] = make_float4(f[0], f[1], f[2], 0.0f);
    rec_tag[it] = make_uint4(live ? (m | (multi ? 0x100u : 0u) | ((unsigned)(ip[2] + off) << 16)) : 0u, (unsigned)a,
                             live ? ((unsigned)(ip[0] + off) | ((unsigned)(ip[1] + off) << 16)) : 0u, __float_as_uint(sw));
    if (!live) return;
    unsigned *const bc = blk_count + g.tile_base;  // tile_base: first block of this grid
    for_each_block_in_reach(g, (float)ip[0] + f[0], (float)ip[1] + f[1], (float)ip[2] + f[2], [&](int bid) { atomicAdd(bc + bid, 1u); });
}

// second pass: the same walk appends (item, mask | multi << 8) to the lists; blk_count counts down to zero.  (Keeping the
// slots of the first pass instead -- no atomics here -- was slower.)
__global__ void __launch_bounds__(128) occ_blk_fill_kernel(const GridDev *__restrict__ grids, int B, long long it0, long long n_items,
                                                           const float4 *__restrict__ rec_pos, const uint4 *__restrict__ rec_tag,
                                                           unsigned *__restrict__ blk_count, const unsigned *__restrict__ blk_start,
                                                           uint2 *__restrict__ blk_ent) {
    const long long it = it0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (it >= it0 + n_items) return;
    const uint4 tg = rec_tag[it];
    if ((tg.x & 0x1ffu) == 0) return;
    const int b = find_grid_item(grids, B, it);
    const GridDev &g = grids[b];
    const float4 f = rec_pos[it];
    const int off = g.cutv + 1;
    const float px = (float)((int)(tg.z & 0xffffu) - off) + f.x, py = (float)((int)(tg.z >> 16) - off) + f.y,
                pz = (float)((int)(tg.x >> 16) - off) + f.z;
    unsigned *const bc = blk_count + g.tile_base;
    const unsigned *const bs = blk_start + g.tile_base;
    const uint2 ent = make_uint2((unsigned)it, tg.x & 0x1ffu);
    uint2 *const be = blk_ent + g.ent_base;
    for_each_block_in_reach(g, px, py, pz, [&](int bid) { be[bs[bid] + atomicSub(bc + bid, 1u) - 1u] = ent; });
}

// compact output: 1 for every block with a candidate list, then an exclusive scan gives its record index
__global__ void occ_blk_flag_kernel(const unsigned *__restrict__ blk_start, long long n_blocks, unsigned *__restrict__ flag) {
    const long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (b <= n_blocks) flag[b] = (b < n_blocks && blk_start[b + 1] != blk_start[b]) ? 1u : 0u;
}

__device__ __forceinline__ void bulk_store_row(float *dst, unsigned src_smem, int bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes) : "memory");
}
__device__ __forceinline__ void store_cmajor_zero(float *grid, int nx, int ny, int nz, int x0, int iy, int iz) {
    if (iy >= ny || iz >= nz) return;
    const long long cs = (long long)nx * ny * nz;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (x0 + k < nx) {
            float *const o = grid + ((long long)(x0 + k) * ny + iy) * nz + iz;
#pragma unroll
            for (int h = 0; h < 8; ++h) __stcs(o + h * cs, 0.0f);
        }
}
// record load through a pinned shared address (ptxas otherwise rebuilds the address from the lane / warp id at the head of every
// run).  Volatile: stays between the __syncwarp()s around the hot loop, i.e. after the stores of the record pass and before
// the next round's.
__device__ __forceinline__ float4 lds_rec4(unsigned a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ void cp_async16(unsigned dst_smem, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src) : "memory");
}
// one 4 x 4 x 8-voxel block (dense [x][y][z][c] tile in shared memory) -> the grid; coordinates (z * 8, y, x, grid); TMA clips
// the part of the box that lies outside the grid
__device__ __forceinline__ void tma_store_block(const CUtensorMap *tm, unsigned src_smem, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%1, %2, %3, %4}], [%5];" ::"l"(tm), "r"(c0), "r"(c1),
                 "r"(c2), "r"(c3), "r"(src_smem)
                 : "memory");
}

#define RG(field) (UNIFORM ? p.u.field : __ldg(&gg->field))
template <bool UNIFORM>
__global__ void __launch_bounds__(R_WARPS * 32, MKB_R_MIN_CTAS) occ_fill_runs_kernel(const RunParams p,
                                                                                     const __grid_constant__ CUtensorMap tmap) {
    __shared__ __align__(128) unsigned char s_raw[R_WARPS][R_WARP_BYTES];
    __shared__ __align__(128) float s_zero[1024];  // one zeroed block (4 KB): the source of every store without atoms in reach

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *const wb = s_raw[warp];
    float4 *const rec = reinterpret_cast<float4 *>(wb);                         // sorted candidates: the four x differences, x lambda
    float4 *const recy = reinterpret_cast<float4 *>(wb + R_CAP * 16);           // (-y lambda, -z lambda, w, tag: mask | flags)
    unsigned char *const msk = wb + R_CAP * 32;                                 // channel mask of the sorted candidate
    unsigned char *const rnk = wb + R_CAP * 33;                                 // rank of a candidate inside its mask bin
    unsigned *const hist = reinterpret_cast<unsigned *>(wb + R_CAP * 34);       // 256 x 16-bit bins in 128 words
    // the hot loop loads through an address the compiler cannot rematerialise (it would rebuild it from S2R SR_TID /
    // SR_CgaCtaId at the head of every run: ten instructions and two slow special-register reads)
    unsigned rec_sa = (unsigned)__cvta_generic_to_shared(wb);
    asm volatile("mov.b32 %0, %0;" : "+r"(rec_sa));
    const unsigned stage_sa = (unsigned)__cvta_generic_to_shared(wb);
    const unsigned zero_sa = (unsigned)__cvta_generic_to_shared(s_zero);

    for (int i = threadIdx.x; i < 1024; i += R_WARPS * 32) s_zero[i] = 0.0f;
    for (int i = lane; i < 128; i += 32) hist[i] = 0u;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const int ly = lane >> 3, lz = lane & 7;
    float fy = (float)ly - 1.5f, fz = (float)lz - 3.5f;  // block frame: origin at the block centre
    // ptxas rebuilds fy / fz from the lane id (SHF, LOP3, I2FP, FADD) at the head of every run instead of keeping two registers
    // alive: an opaque move pins them (8 instructions per run, 3 % of the kernel)
    asm volatile("mov.b32 %0, %0;" : "+f"(fy));
    asm volatile("mov.b32 %0, %0;" : "+f"(fz));
    const float INF = __int_as_float(0x7f800000);
    bool pending = false;  // lanes 0..15: bulk copies still reading the stage
    // lambda = 2^64 / cut (voxel units): d2 == cut2 lands on 2^128, the float overflow threshold
    // The FLOAT is the root value and the double its exact image: with lamf = (float)lam ptxas kept only the double and
    // re-converted it (F2F.F32.F64, a slow-pipe instruction the first FFMA then waits for) at the head of EVERY hot-loop trip.
    // Atoms and voxels are scaled by the same number this way; cwf = 2^64 / lambda (= cut up to 6e-8) keeps r = U w exact.
    float lamf = UNIFORM ? (float)(18446744073709551616.0 / sqrt((double)p.u.cut2v)) : 0.0f;
    asm volatile("mov.b32 %0, %0;" : "+f"(lamf));
    double lam = (double)lamf;
    float cwf = UNIFORM ? (float)(18446744073709551616.0 / lam) : 0.0f;

    for (;;) {
        unsigned id = 0;
        if (lane == 0) id = atomicAdd(p.queue, 1u);
        id = __shfl_sync(0xffffffffu, id, 0);
        if (id >= p.total_items) break;
        // ---- decode the item: grid, (x, y) block column, chunk of R_ZC z blocks
        int gi;
        unsigned local;
        if (UNIFORM) {
            gi = (int)(id / p.u_ipg);
            local = id - (unsigned)gi * p.u_ipg;
        } else {
            const long long gid = (long long)id + p.item0;
            int lo = 0, hi = p.B - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (__ldg(p.item_base + mid) <= gid) lo = mid; else hi = mid - 1;
            }
            gi = lo;
            local = (unsigned)(gid - __ldg(p.item_base + gi));
        }
        const GridDev *gg = p.grids + gi;
        const int nx = RG(dims[0]), ny = RG(dims[1]), nz = RG(dims[2]);
        const int nbz = (nz + R_BZ - 1) / R_BZ;
        const unsigned nby = UNIFORM ? p.u_nby : (unsigned)(ny + 3) >> 2, nzc = UNIFORM ? p.u_nzc : (unsigned)(nbz + p.zc - 1) / p.zc;
        const int zc = (int)(local % nzc);
        const unsigned bxy = local / nzc;
        const int byi = (int)(bxy % nby), bxi = (int)(bxy / nby);
        const int x0 = bxi * 4, y0 = byi * 4;
        const long long out_offset = UNIFORM ? p.u.out_offset + (long long)gi * p.u_out_stride : __ldg(&gg->out_offset);
        // output rows of a block: lane (< 16) -> (x = lane >> 2, y = lane & 3), 8 voxels x 8 channels = 256 B each
        const int rix = x0 + (lane >> 2), riy = y0 + (lane & 3);
        const bool row_ok = lane < 16 && rix < nx && riy < ny;
        float *const row_base = p.out + (out_offset + ((long long)rix * ny + riy) * nz) * 8;
        const float cut2 = RG(cut2v);
        const int off = RG(cutv) + 1;
        const int bz_begin = zc * p.zc, bz_end = min(nbz, bz_begin + p.zc);
        // candidate list offsets of the item's blocks (consecutive block ids): lanes 0..R_ZC
        const long long blk0 = (UNIFORM ? p.u.tile_base + (long long)gi * p.u_bpg : __ldg(&gg->tile_base)) + (long long)bxy * nbz + bz_begin;
        const unsigned my_start = __ldg(p.blk_start + blk0 + min(lane, bz_end - bz_begin));
        if (__shfl_sync(0xffffffffu, my_start, bz_end - bz_begin) == __shfl_sync(0xffffffffu, my_start, 0)) {
            // no atom reaches any block of the item: one bulk copy of zeros per output row (TMA, nothing to wait for)
            const int z0 = bz_begin * R_BZ;
            if (p.blk_rank) {
            } else if (p.cmajor) {
                for (int bzi = bz_begin; bzi < bz_end; ++bzi) store_cmajor_zero(p.out + out_offset * 8, nx, ny, nz, x0, y0 + ly, bzi * R_BZ + lz);
            } else if (p.use_tmap) {
                if (lane == 0) {
                    for (int bzi = bz_begin; bzi < bz_end; ++bzi) tma_store_block(&tmap, zero_sa, bzi * (R_BZ * 8), y0, x0, gi);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            } else {
                if (row_ok) bulk_store_row(row_base + z0 * 8, zero_sa, (min(nz, bz_end * R_BZ) - z0) * 32);
                if (lane < 16) asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            continue;
        }

        if (!UNIFORM) {
            lamf = (float)(18446744073709551616.0 / sqrt((double)cut2));
            lam = (double)lamf;
            cwf = (float)(18446744073709551616.0 / lam);
        }
        for (int bzi = bz_begin; bzi < bz_end; ++bzi) {
            const int z0 = bzi * R_BZ;
            const int row_bytes = min(R_BZ, nz - z0) * 32;
            float *const row_dst = row_base + z0 * 8;
            const unsigned ls = __shfl_sync(0xffffffffu, my_start, bzi - bz_begin);
            const unsigned n = __shfl_sync(0xffffffffu, my_start, bzi - bz_begin + 1) - ls;
            if (n == 0) {
                if (p.blk_rank) {
                } else if (p.cmajor) {
                    store_cmajor_zero(p.out + out_offset * 8, nx, ny, nz, x0, y0 + ly, z0 + lz);
                } else if (p.use_tmap) {
                    if (lane == 0) {
                        tma_store_block(&tmap, zero_sa, z0 * 8, y0, x0, gi);
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                } else {
                    if (row_ok) bulk_store_row(row_dst, zero_sa, row_bytes);
                    if (lane < 16) asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                continue;
            }

            float acc[8][4];
#pragma unroll
            for (int h = 0; h < 8; ++h)
#pragma unroll
                for (int k = 0; k < 4; ++k) acc[h][k] = INF;
            // lattice point of the block corner in the records' offset frame
            const int cx = x0 + off, cy = y0 + off, cz = z0 + off;

            for (unsigned base = 0; base < n; base += R_CAP) {
                const int np = (int)min((unsigned)R_CAP, n - base);
                const uint2 *const ent = p.blk_ent + ls + base;
                // ---- pass 1: histogram of the channel masks, rank of every candidate inside its bin
                unsigned ey[R_CAP / 32];
                {
#pragma unroll
                    for (int u = 0; u < R_CAP / 32; ++u) {  // all loads of the round in flight together
                        const int j = u * 32 + lane;
                        ey[u] = j < np ? __ldg(&ent[j].y) : 0u;
                    }
                }
                // the histogram trips carry no other code: the per-channel path of multi-sigma atoms (rare: user float channels) used
                // to be inlined in each of the R_CAP / 32 unrolled trips -- 34 KB of code that the instruction cache had to skip
                bool any_multi = false;
#pragma unroll
                for (int u = 0; u < R_CAP / 32; ++u) {
                    const int j0 = u * 32;
                    if (j0 >= np) break;
                    const int j = j0 + lane;
                    const uint2 e = make_uint2(0u, ey[u]);
                    const bool multi = (e.y & 0x100u) != 0;
                    any_multi |= multi;
                    if (j < np) {
                        const unsigned m = multi ? 0u : (e.y & 255u), sh = (m & 1u) * 16u;
                        const unsigned old = atomicAdd(&hist[m >> 1], 1u << sh);
                        rnk[j] = (unsigned char)((old >> sh) & 0xffffu);
                    }
                }
                if (__any_sync(0xffffffffu, any_multi)) {
#pragma unroll 1
                    for (int j0 = 0; j0 < np; j0 += 32) {
                        const int j = j0 + lane;
                        const uint2 e = j < np ? __ldg(ent + j) : make_uint2(0u, 0u);
                        const bool multi = (e.y & 0x100u) != 0;
                    // atoms with several distinct sigmas (user float channels): whole-warp per-channel path; they stay in
                        // the list under mask 0 (a run that updates no channel)
                        for (unsigned bm = __ballot_sync(0xffffffffu, multi); bm; bm &= bm - 1) {
                            const unsigned it = __shfl_sync(0xffffffffu, e.x, __ffs(bm) - 1);
                            const float4 f = __ldg(p.rec_pos + it);
                            const uint4 tg = __ldg(p.rec_tag + it);
                            const float ax = (float)((int)(tg.z & 0xffffu) - cx) + (f.x - 1.5f), ay = (float)((int)(tg.z >> 16) - cy) + (f.y - 1.5f),
                                        az = (float)((int)(tg.x >> 16) - cz) + (f.z - 3.5f);
                            const float dy = ay - fy, dz = az - fz;
                            const float s2 = fmaf(dz, dz, dy * dy);
                            const double ivs = RG(inv_vs);
                            float d2[4];
#pragma unroll
                            for (int k2 = 0; k2 < 4; ++k2) {
                                const float dx = ax - ((float)k2 - 1.5f);
                                d2[k2] = fmaf(dx, dx, s2);
                            }
#pragma unroll
                            for (int h = 0; h < 8; ++h) {
                                const double sv = __ldg(p.sigmas + (long long)tg.y * 8 + h) * ivs;
                                if (sv == 0.0 || sv != sv) continue;
                                const float w = (float)(1.0 / (sv * sv));
#pragma unroll
                                for (int k2 = 0; k2 < 4; ++k2)
                                    if (d2[k2] < cut2) acc[h][k2] = fminf(acc[h][k2], d2[k2] * w);
                            }
                        }
                    }
                }
                __syncwarp();
                // ---- counting sort by channel mask: END offsets of the 256 bins (8 per lane); a candidate of rank r in its
                // bin goes to end - 1 - r, so the rank-0 candidate closes the run
                {
                    unsigned cnt[8], off8[8];
                    const uint4 hw = *reinterpret_cast<const uint4 *>(hist + 4 * lane);
                    cnt[0] = hw.x & 0xffffu; cnt[1] = hw.x >> 16; cnt[2] = hw.y & 0xffffu; cnt[3] = hw.y >> 16;
                    cnt[4] = hw.z & 0xffffu; cnt[5] = hw.z >> 16; cnt[6] = hw.w & 0xffffu; cnt[7] = hw.w >> 16;
                    unsigned sum = 0;
#pragma unroll
                    for (int j = 0; j < 8; ++j) { sum += cnt[j]; off8[j] = sum; }
                    unsigned v = sum;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned t = __shfl_up_sync(0xffffffffu, v, o);
                        if (lane >= o) v += t;
                    }
                    const unsigned excl = v - sum;
#pragma unroll
                    for (int j = 0; j < 8; ++j) off8[j] += excl;
                    *reinterpret_cast<uint4 *>(hist + 4 * lane) =
                        make_uint4(off8[0] | (off8[1] << 16), off8[2] | (off8[3] << 16), off8[4] | (off8[5] << 16), off8[6] | (off8[7] << 16));
                }
                // the stage of the previous block aliases the records: its bulk copies must have read it
                if (pending) {
                    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    pending = false;
                }
                __syncwarp();
                // ---- pass 2: records in run order, scaled by lambda (float64 rebase: one rounding per coordinate); the tag of the
                // record that closes a run carries the run's mask and the flags of the run loop.
                // sub-pass a: the raw per-atom data of every candidate goes straight to its sorted slot (cp.async, all in flight)
                for (int j = lane; j < np; j += 32) {
                    const uint2 e = __ldg(ent + j);
                    const unsigned m = (e.y & 0x100u) ? 0u : (e.y & 255u);
                    const unsigned pos = ((hist[m >> 1] >> ((m & 1u) * 16u)) & 0xffffu) - 1u - (unsigned)rnk[j];
                    cp_async16(rec_sa + 16u * pos, p.rec_pos + e.x);
                    cp_async16(rec_sa + (unsigned)(R_CAP * 16) + 16u * pos, p.rec_tag + e.x);
                    msk[pos] = (unsigned char)m;
                }
                asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
                __syncwarp();
                // sub-pass b: slot by slot in place (a lane reads and writes its own slots only)
                for (int j = lane; j < np; j += 32) {
                    const unsigned pos = (unsigned)j;
                    const unsigned m = msk[pos];
                    const unsigned rk = (((hist[m >> 1] >> ((m & 1u) * 16u)) & 0xffffu) - 1u == pos) ? 0u : 1u;  // 0: closes its run
                    const float4 f = rec[pos];
                    const uint4 tg = *reinterpret_cast<const uint4 *>(recy + pos);
                    const float sw = __uint_as_float(tg.w);  // 1 / sigma (voxel units)
                    const double ex = (double)((int)(tg.z & 0xffffu) - cx) + ((double)f.x - 1.5);
                    const double ey = (double)((int)(tg.z >> 16) - cy) + ((double)f.y - 1.5);
                    const double ez = (double)((int)(tg.x >> 16) - cz) + ((double)f.z - 3.5);
                    const float xs = (float)(ex * lam);
                    rec[pos] = make_float4(fmaf(-1.5f, lamf, -xs), fmaf(-0.5f, lamf, -xs), fmaf(0.5f, lamf, -xs), fmaf(1.5f, lamf, -xs));
                    const float wh = (sw * cwf) * 5.421010862427522e-20f;  // (cut / sigma) 2^-64
                    const float wt = wh * wh;                              // w = 1 / (sigma lambda)^2
                    // tag: mask | bit 8: the run also closes its group (no candidate in the bins m + 1 .. m | 15; hist holds END
                    // offsets) | bit 9: last record of the round | bit 31: the record closes its run
                    const unsigned mh = m | 15u;
                    const unsigned e0 = (hist[m >> 1] >> ((m & 1u) * 16u)) & 0xffffu, e1 = (hist[mh >> 1] >> 16) & 0xffffu;
                    recy[pos] = make_float4(-(float)(ey * lam), -(float)(ez * lam), wt,
                                            __uint_as_float(m | ((rk == 0 && e0 == e1) ? 0x100u : 0u) | (rk == 0 ? 0x80000000u : 0u) |
                                                            (pos + 1u == (unsigned)np ? 0x200u : 0u)));
                }
                __syncwarp();
                *reinterpret_cast<uint4 *>(hist + 4 * lane) = make_uint4(0u, 0u, 0u, 0u);
                __syncwarp();

                // ---- the hot loop: one warp-uniform candidate per half trip, 4 voxels per lane; two records in flight
                // (a / b ping-pong, the next one is loaded before the current one is evaluated)
                {
#define MKB_LDREC(I) lds_rec4(rec_sa + 16u * (unsigned)(I))
#define MKB_LDRECY(I) lds_rec4(rec_sa + (unsigned)(R_CAP * 16) + 16u * (unsigned)(I))
#define MKB_RUN_R2(D, Y, R)                                                                       \
    float R##0, R##1, R##2, R##3;                                                                 \
    {                                                                                             \
        const float dy_ = fmaf(fy, lamf, Y.x), dz_ = fmaf(fz, lamf, Y.y);                         \
        const float s2_ = __fadd_rn(__fmul_rn(dy_, dy_), __fmul_rn(dz_, dz_));                    \
        R##0 = __fmul_rn(fmaf(D.x, D.x, s2_), Y.z);                                               \
        R##1 = __fmul_rn(fmaf(D.y, D.y, s2_), Y.z);                                               \
        R##2 = __fmul_rn(fmaf(D.z, D.z, s2_), Y.z);                                               \
        R##3 = __fmul_rn(fmaf(D.w, D.w, s2_), Y.z);                                               \
    }
                    float4 a = MKB_LDREC(0), ya = MKB_LDRECY(0);
                    int i = 1;  // next record to load; i == np reads past the list (inside this warp's buffer), never used
                    float M0 = INF, M1 = INF, M2 = INF, M3 = INF;
                    // one trip per run; bit 9 of the tag marks the last record of the round (ptxas otherwise rebuilds the candidate
                    // count for a compare at the end of every run)
#pragma unroll 1
                    for (bool more = true; more;) {
                        float m0 = INF, m1 = INF, m2 = INF, m3 = INF;
                        unsigned mask;
#pragma unroll 1
                        for (;;) {
                            const float4 b = MKB_LDREC(i), yb = MKB_LDRECY(i);
                            MKB_RUN_R2(a, ya, ra)
                            if (__float_as_int(ya.w) < 0) {  // the tag of the record that closes a run has its sign bit set (warp-uniform)
                                m0 = fminf(m0, ra0); m1 = fminf(m1, ra1); m2 = fminf(m2, ra2); m3 = fminf(m3, ra3);
                                mask = __float_as_uint(ya.w);  // mask | close-the-group << 8 | last-of-the-round << 9
                                a = b;
                                ya = yb;
                                i += 1;
                                break;
                            }
                            a = MKB_LDREC(i + 1);
                            ya = MKB_LDRECY(i + 1);
                            MKB_RUN_R2(b, yb, rb)
                            m0 = fminf(fminf(m0, ra0), rb0); m1 = fminf(fminf(m1, ra1), rb1);
                            m2 = fminf(fminf(m2, ra2), rb2); m3 = fminf(fminf(m3, ra3), rb3);
                            i += 2;
                            if (__float_as_int(yb.w) < 0) {
                                mask = __float_as_uint(yb.w);
                                break;
                            }
                        }
#pragma unroll
                        for (int h = 0; h < 4; ++h)
                            if (mask & (1u << h)) {
                                acc[h][0] = fminf(acc[h][0], m0); acc[h][1] = fminf(acc[h][1], m1);
                                acc[h][2] = fminf(acc[h][2], m2); acc[h][3] = fminf(acc[h][3], m3);
                            }
                        M0 = fminf(M0, m0); M1 = fminf(M1, m1); M2 = fminf(M2, m2); M3 = fminf(M3, m3);
                        if (mask & 0x100u) {  // warp-uniform: the group of runs sharing this high nibble ends here
#pragma unroll
                            for (int h = 4; h < 8; ++h)
                                if (mask & (1u << h)) {
                                    acc[h][0] = fminf(acc[h][0], M0); acc[h][1] = fminf(acc[h][1], M1);
                                    acc[h][2] = fminf(acc[h][2], M2); acc[h][3] = fminf(acc[h][3], M3);
                                }
                            M0 = INF; M1 = INF; M2 = INF; M3 = INF;
                        }
                        more = (mask & 0x200u) == 0u;
                    }
#undef MKB_RUN_R2
#undef MKB_LDREC
#undef MKB_LDRECY
                }
                __syncwarp();
            }

            // ---- epilogue: value = 1 - exp(-(1/r)^6) once per voxel-channel.  The minima go to the stage (output layout:
            // voxel-major, 8 channels = two float4) as they are; a compact loop then turns r into the value in place, 4
            // channels per lane and trip (an epilogue unrolled over the 32 accumulators was 10 KB of code: with 28 warps in
            // different phases the instruction cache did not hold it).
            if (pending) {
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                pending = false;
            }
            __syncwarp();
            float4 *const stage = reinterpret_cast<float4 *>(wb);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int v = ((k * 4 + ly) * 8 + lz) * 2;
                stage[v] = make_float4(acc[0][k], acc[1][k], acc[2][k], acc[3][k]);
                stage[v + 1] = make_float4(acc[4][k], acc[5][k], acc[6][k], acc[7][k]);
            }
            __syncwarp();
#pragma unroll 1
            for (int it = 0; it < 8; ++it) {
                float4 v = stage[it * 32 + lane];
                const float LIVE = 0.5f * R_GATE_HUGE;  // r of a voxel-channel no atom reached: +inf
                const bool live = fminf(fminf(v.x, v.y), fminf(v.z, v.w)) < LIVE;
                if (__any_sync(0xffffffffu, live)) {
                    v.x = occ_value(rcp_approx(v.x)); v.y = occ_value(rcp_approx(v.y));
                    v.z = occ_value(rcp_approx(v.z)); v.w = occ_value(rcp_approx(v.w));
                } else {
                    v = make_float4(0.f, 0.f, 0.f, 0.f);
                }
                stage[it * 32 + lane] = v;
            }
            if (p.cmajor) {  // channel-major grid: 8 lanes = one 32-byte segment per (channel, x, y)
                __syncwarp();
                const long long cs = (long long)nx * ny * nz;
                if (y0 + ly < ny && z0 + lz < nz) {
#pragma unroll 1
                    for (int k = 0; k < 4; ++k)
                        if (x0 + k < nx) {
                            const int v = ((k * 4 + ly) * 8 + lz) * 2;
                            const float4 lo4 = stage[v], hi4 = stage[v + 1];
                            float *const o = p.out + out_offset * 8 + ((long long)(x0 + k) * ny + (y0 + ly)) * nz + (z0 + lz);
                            __stcs(o, lo4.x); __stcs(o + cs, lo4.y); __stcs(o + 2 * cs, lo4.z); __stcs(o + 3 * cs, lo4.w);
                            __stcs(o + 4 * cs, hi4.x); __stcs(o + 5 * cs, hi4.y); __stcs(o + 6 * cs, hi4.z); __stcs(o + 7 * cs, hi4.w);
                        }
                }
                __syncwarp();  // the stage is the next block's record buffer
                continue;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (p.blk_rank && !p.sparse_dense) {  // compact output: the whole 4 KB stage is one record, one bulk copy
                if (lane == 0) bulk_store_row(p.out + 1024ll * __ldg(p.blk_rank + blk0 + (bzi - bz_begin)), stage_sa, 4096);
            } else if (p.use_tmap) {
                if (lane == 0) tma_store_block(&tmap, stage_sa, z0 * 8, y0, x0, gi);
            } else if (row_ok) bulk_store_row(row_dst, stage_sa + lane * 256, row_bytes);
            if (lane < 16) asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            pending = true;
        }
    }
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the copies
}
#undef RG

// ---------------------------------------------------------------------------------------------------------
// Gate band pre-pass.  One thread per atom item walks the (y, z) lattice rows of the atom's cutoff sphere.  A row crosses
// the sphere at x = px -+ sqrt(cut2 - s); only the lattice point nearest to a crossing can lie within the band
// |d2 - cut2| <= band.  Such voxels get a bit in `bitmap` (bit = voxel index in the dense batch order); the first thread
// to set a bit also appends the voxel to `list` (fix[0] = count, capacity `cap`: beyond it occ_fix_scan_kernel takes over).
// ---------------------------------------------------------------------------------------------------------
constexpr float R_FIND_BAND = 2.0e-6f;  // relative; fill error (< 1e-6, see DESIGN.md) + this kernel's own float32 error
constexpr int FIX_HDR = 4;              // words in front of the list: count

__global__ void __launch_bounds__(128) occ_band_kernel(const float *__restrict__ coords, const GridDev *__restrict__ grids, int B,
                                                       long long n_items, unsigned *__restrict__ bitmap,
                                                       unsigned long long *__restrict__ fix, unsigned cap) {
    const long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (it >= n_items) return;
    const int b = find_grid_item(grids, B, it);
    const GridDev &g = grids[b];
    const long long a = g.atom_begin + (it - g.item_base);
    int ip[3];
    float f[3];
    bool live = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double pv = ((double)coords[3 * a + d] - g.origin[d]) * g.inv_vs;
        live = live && (pv >= -(double)g.cutv - 1.0) && (pv <= (double)(g.dims[d] + g.cutv));
        const double r = live ? rint(pv) : 0.0;
        ip[d] = (int)r;
        f[d] = (float)(pv - r);
    }
    if (!live) return;  // NaN or out of reach of every voxel
    const float cut2 = g.cut2v;
    const float band = R_FIND_BAND * cut2;
    const int W = (int)(sqrtf(cut2) + 0.5f) + 1;  // |j - f| <= cut with |f| <= 0.5 (+1: rounding slack)
    const float RND = 12582912.0f;                  // 1.5 * 2^23: (x + RND) - RND == rint(x) for |x| < 2^22
    const int ny = g.dims[1], nz = g.dims[2];
    for (int jy = -W; jy <= W; ++jy) {
        const int iy = ip[1] + jy;
        const float dy = (float)jy - f[1];
        const float A = fmaf(-dy, dy, cut2);
        if (A < -band || iy < 0 || iy >= ny) continue;
        // z rows that can cross the sphere: |jz - f_z| <= sqrt(A + band) (a superset; the exact test follows per row)
        const float zr = sqrtf(A + band) + 1e-3f;
        const int jz_lo = max(-W, (int)ceilf(f[2] - zr)), jz_hi = min(W, (int)floorf(f[2] + zr));
        for (int jz = jz_lo; jz <= jz_hi; ++jz) {
            const float dz = (float)jz - f[2];
            const float h2 = fmaf(-dz, dz, A);  // cut2 - s
            if (h2 < -band) continue;           // the row misses the sphere
            const float hp = fmaxf(h2, 0.0f);
            const float hh = hp * rsqrtf(fmaxf(hp, 1e-30f));
            const float jxa = (f[0] + hh + RND) - RND, jxb = (f[0] - hh + RND) - RND;
            const float da = jxa - f[0], db = jxb - f[0];
            const float ta = fmaf(da, da, -h2), tb = fmaf(db, db, -h2);
            const bool fa = fabsf(ta) <= band, fb = (fabsf(tb) <= band) & (jxb != jxa);
            if (fa | fb) {
                const int iz = ip[2] + jz;
                if (iz < 0 || iz >= nz) continue;
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    if (q == 0 ? !fa : !fb) continue;
                    const int ix = ip[0] + (int)(q == 0 ? jxa : jxb);
                    if (ix < 0 || ix >= g.dims[0]) continue;
                    const long long v = g.vox_base + (((long long)ix * ny + iy) * nz + iz);
                    const unsigned bit = 1u << (v & 31);
                    const unsigned old = atomicOr(bitmap + (v >> 5), bit);
                    if (!(old & bit)) {
                        const unsigned long long slot = atomicAdd(fix, 1ull);
                        if (slot < cap) fix[FIX_HDR + slot] = (unsigned long long)v;
                    }
                }
            }
        }
    }
}

// float64 re-evaluation of one voxel with the reference's operations (pyx:46-61): d2 as the reference computes it
// (centres fl(fl(i*vs) + origin), voxeldescriptors.py:125-132,245), max of sigma^2/d2 per channel, 1 - exp(-q^6).
// One warp per flagged voxel; the atoms are those of the voxel's block list.
__device__ __forceinline__ void occ_fix_voxel(const GridDev *__restrict__ grids, int B, long long v, int lane,
                                              const float *__restrict__ coords, const double *__restrict__ sigmas,
                                              const double *__restrict__ radii, const unsigned *__restrict__ chanmask,
                                              const uint4 *__restrict__ rec_tag, const unsigned *__restrict__ blk_start,
                                              const uint2 *__restrict__ blk_ent, float *__restrict__ out, int cmajor,
                                              const unsigned *__restrict__ blk_rank) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (grids[mid].vox_base <= v) lo = mid; else hi = mid - 1;
    }
    const GridDev *g = grids + lo;
    const long long lv = v - g->vox_base;
    const int nz = g->dims[2], ny = g->dims[1];
    const int iz = (int)(lv % nz), iy = (int)((lv / nz) % ny), ix = (int)(lv / ((long long)nz * ny));
    const int nby = (ny + 3) >> 2, nbz = (nz + R_BZ - 1) / R_BZ;
    const long long bid = g->tile_base + ((long long)(ix >> 2) * nby + (iy >> 2)) * nbz + iz / R_BZ;
    const unsigned e0 = __ldg(blk_start + bid), e1 = __ldg(blk_start + bid + 1);
    const double cx = __dadd_rn(__dmul_rn((double)ix, g->vs), g->origin[0]);
    const double cy = __dadd_rn(__dmul_rn((double)iy, g->vs), g->origin[1]);
    const double cz = __dadd_rn(__dmul_rn((double)iz, g->vs), g->origin[2]);
    double q[8];
#pragma unroll
    for (int h = 0; h < 8; ++h) q[h] = 0.0;
    for (unsigned i = e0 + lane; i < e1; i += 32) {
        const unsigned a = __ldg(&rec_tag[__ldg(&blk_ent[g->ent_base + i].x)].y);
        const double dx = (double)coords[3ll * a + 0] - cx;
        const double dy = (double)coords[3ll * a + 1] - cy;
        const double dz = (double)coords[3ll * a + 2] - cz;
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (!(d2 < CUTOFF_A * CUTOFF_A)) continue;
#pragma unroll
        for (int h = 0; h < 8; ++h) {
            double s;
            if (sigmas) s = sigmas[(long long)a * 8 + h];
            else s = ((chanmask[a] >> h) & 1u) ? radii[a] : 0.0;
            if (s == 0.0 || s != s) continue;
            const double qq = (s * s) / d2;  // +inf at d2 == 0 -> value 1 (pyx:57)
            q[h] = qq > q[h] ? qq : q[h];
        }
    }
#pragma unroll
    for (int h = 0; h < 8; ++h)
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double t = __shfl_xor_sync(0xffffffffu, q[h], o);
            q[h] = t > q[h] ? t : q[h];
        }
    double mq = q[0];
#pragma unroll
    for (int h = 1; h < 8; ++h) mq = (lane == h) ? q[h] : mq;
    if (lane < 8) {
        const double q3 = mq * mq * mq;
        const float val = (float)(-expm1(-(q3 * q3)));
        if (blk_rank) out[1024ll * __ldg(blk_rank + bid) + ((((ix & 3) * 4 + (iy & 3)) * 8 + (iz & 7)) * 8) + lane] = val;
        else if (cmajor) out[g->out_offset * 8 + (long long)lane * ((long long)g->dims[0] * ny * nz) + lv] = val;
        else out[(g->out_offset + lv) * 8 + lane] = val;
    }
}

__global__ void __launch_bounds__(256) occ_fix_list_kernel(const GridDev *__restrict__ grids, int B,
                                                           const unsigned long long *__restrict__ fix, unsigned cap,
                                                           const float *__restrict__ coords, const double *__restrict__ sigmas,
                                                           const double *__restrict__ radii, const unsigned *__restrict__ chanmask,
                                                           const uint4 *__restrict__ rec_tag, const unsigned *__restrict__ blk_start,
                                                           const uint2 *__restrict__ blk_ent, float *__restrict__ out, int cmajor,
                                                           const unsigned *__restrict__ blk_rank) {
    const unsigned long long n = fix[0];
    if (n > cap) return;  // the list overflowed: occ_fix_scan_kernel walks the bitmap instead
    const int lane = threadIdx.x & 31;
    const unsigned nw = (gridDim.x * blockDim.x) >> 5;
    for (unsigned long long w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n; w += nw)
        occ_fix_voxel(grids, B, (long long)fix[FIX_HDR + w], lane, coords, sigmas, radii, chanmask, rec_tag, blk_start, blk_ent, out, cmajor, blk_rank);
}

__global__ void __launch_bounds__(256) occ_fix_scan_kernel(const GridDev *__restrict__ grids, int B, long long n_words,
                                                           const unsigned *__restrict__ bitmap,
                                                           const unsigned long long *__restrict__ fix, unsigned cap,
                                                           const float *__restrict__ coords, const double *__restrict__ sigmas,
                                                           const double *__restrict__ radii, const unsigned *__restrict__ chanmask,
                                                           const uint4 *__restrict__ rec_tag, const unsigned *__restrict__ blk_start,
                                                           const uint2 *__restrict__ blk_ent, float *__restrict__ out, int cmajor,
                                                           const unsigned *__restrict__ blk_rank) {
    if (fix[0] <= cap) return;
    const int lane = threadIdx.x & 31;
    const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long w0 = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; w0 < n_words; w0 += nw * 32) {
        const unsigned mine = (w0 + lane < n_words) ? __ldg(bitmap + w0 + lane) : 0u;
        for (unsigned wm = __ballot_sync(0xffffffffu, mine != 0); wm; wm &= wm - 1) {
            const int wl = __ffs(wm) - 1;
            for (unsigned bits = __shfl_sync(0xffffffffu, mine, wl); bits; bits &= bits - 1)
                occ_fix_voxel(grids, B, ((w0 + wl) << 5) + (__ffs(bits) - 1), lane, coords, sigmas, radii, chanmask, rec_tag,
                              blk_start, blk_ent, out, cmajor, blk_rank);
        }
    }
}

}  // namespace mkb
