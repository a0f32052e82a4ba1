/*
 * mkb200.h -- C-ABI of libmkb200.so: the H100-native voxel-occupancy and trajectory-distance engine.
 *
 * This is the drop-in boundary for ONE hot path of Acellera/moleculekit (SURVEY.md section 8):
 *   moleculekit/occupancy_utils/occupancy_utils.pyx   (calculate_occupancy)
 *   moleculekit/distance_utils/distance_utils.pyx     (dist_trajectory, contacts_trajectory,
 *                                                      dist_trajectory_reduction[_pairs], cdist, pdist,
 *                                                      squareform, get_collisions)
 * The reference exposes these as Cython `def` functions over numpy memoryviews (no C header); each entry
 * point below cites the reference function it replaces.  Conventions:
 *   - plain C types only: pointers, sizes, scalars.  No torch / numpy types.
 *   - bulk arrays are DEVICE pointers (the Python host obtains them from torch.Tensor.data_ptr());
 *     small per-grid descriptors are HOST arrays (they size the launch); `stream` is a cudaStream_t
 *     passed as void* (0 = legacy default stream).  All work is stream-ordered; nothing blocks the host
 *     except where stated (mkb_contacts_count returns a host total).
 *   - every function returns MKB_OK (0) or a negative mkb_status; mkb_last_error(h) gives the message.
 *   - the caller owns every input/output array; the handle owns only scratch (cell lists, scan temp),
 *     grown on demand and freed by mkb_destroy.  One handle per device; not thread-safe per handle.
 *   - there is NO CPU fallback: without a CUDA device mkb_create fails with MKB_ERR_CUDA.
 */
#ifndef MKB200_H
#define MKB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MKB_VERSION 100 /* 0.1.0 */

typedef enum {
    MKB_OK = 0,
    MKB_ERR_BAD_ARG = -1,
    MKB_ERR_CUDA = -2,
    MKB_ERR_NOMEM = -3,
    MKB_ERR_CAPACITY = -4,
    MKB_ERR_UNSUPPORTED = -5 /* a valid request this entry point cannot serve (e.g. compact output outside its domain) */
} mkb_status;

typedef struct mkb_ctx *mkb_handle_t;

/* flags for the occupancy entry points */
#define MKB_OCC_ACCUMULATE 1u /* out = value if value > out, as the reference accumulates into the caller's buffer
                                 (occupancy_utils.pyx:56-61): only voxel-channels that some atom with a non-zero sigma
                                 reaches within 5 A are updated; the others keep their bits (a negative, -inf or NaN
                                 prefill included), and NaN in `out` sticks.  Without it `out` is overwritten (caller
                                 passes zeros, voxeldescriptors.py:531, so both agree) */
#define MKB_OCC_LAYOUT_CXYZ 2u /* SURVEY 8f row 1: grid b is written channel-major, out[b] = float32 [C][nx][ny][nz]
                                 (the layout a Conv3d consumer wants, instead of the reference's [nx][ny][nz][C]
                                 reshaped view, voxeldescriptors.py:298-299); grid b still starts at out + out_offset*C.
                                 Same values bit for bit.  mkb_occupancy_grid_batch only. */

/* output modes of the distance entry points (host post-ops of projections/util.py:74-84 fused in) */
#define MKB_DIST_DISTANCES 0 /* float32 distances, optionally truncated */
#define MKB_DIST_CONTACTS 1  /* uint8 (bool) = distance <= threshold, after optional truncate */
#define MKB_DIST_DISTANCES_FAST 4 /* float32 distances within 4 ulp of the reference's float32 sequence (the reference's
                                     minimum-image roundings, fused sum of squares, approximate square root); same NaN
                                     pattern; BASELINE north star asks for 1e-5 relative.  mkb_dist_trajectory only. */

int mkb_version(void);
int mkb_create(int device, mkb_handle_t *out);
int mkb_destroy(mkb_handle_t h);
const char *mkb_last_error(mkb_handle_t h);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t mkb_launch_count(mkb_handle_t h);
/* Per-kernel device timing for the roofline report: when on, the occupancy and distance entry points record CUDA
 * events on the launch stream before their preparation kernels, before the main kernel and after it.
 * mkb_get_timing synchronises on the last event and returns the two intervals of the most recent call (ms). */
int mkb_set_timing(mkb_handle_t h, int on);
int mkb_get_timing(mkb_handle_t h, float *prep_ms, float *main_ms);
/* name of the main kernel the most recent occupancy / distance entry point launched (static string; "" before any call) */
const char *mkb_last_kernel(mkb_handle_t h);

/* One regular voxel grid: centre of voxel (ix,iy,iz) = fl(fl(i*voxelsize) + origin[d]) in float64, exactly
 * as moleculekit/tools/voxeldescriptors.py:125-132,245 builds `centers`; flat voxel index
 * (ix*ny + iy)*nz + iz (z fastest), channels minor. */
typedef struct {
    double origin[3];   /* bb_min of getCenters (voxeldescriptors.py:231-243) */
    double voxelsize;   /* isotropic voxel edge, Angstrom */
    int32_t dims[3];    /* nx, ny, nz */
    int32_t reserved;
    int64_t atom_begin; /* rows [atom_begin, atom_end) of coords/sigmas belong to this grid */
    int64_t atom_end;
    int64_t out_offset; /* first voxel of this grid in `out`, in voxels (row = C floats) */
} mkb_grid_desc;

/* K1+K2: batched occupancy on regular grids.
 * Replaces calculate_occupancy (occupancy_utils.pyx:34-61) + the centre materialisation of getCenters for every
 * grid of the batch in one launch sequence (bin atoms -> scan -> scatter -> fill).
 *   coords  [n_atoms,3] float32 device      (reference: coords f32[:,:])
 *   sigmas  [n_atoms,C] float64 device      (reference: sigmas f64[:,:]; 0 = channel off, NaN ignored)
 *   grids   [B] HOST descriptors
 *   out     [sum_b nx*ny*nz, C] float32 device (the reference's float64 results; the host wrapper upcasts)
 * 1 <= C <= 32. */
int mkb_occupancy_grid_batch(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                             int64_t n_atoms, int32_t C, const mkb_grid_desc *grids, int32_t B,
                             float *out, uint32_t flags);

/* K1 with device-side channel assembly (SURVEY 8f row 1): the reference builds sigmas = vdw_radius[:, None] *
 * channels.astype(float) on the host (voxeldescriptors.py:332-335); here the (n_atoms,) float64 radii and a per-atom
 * channel bit mask (bit c set = atom belongs to channel c) are the inputs and the (n_atoms, C) float64 matrix never
 * exists -- 12 instead of 8*C bytes per atom over PCIe.  Bit-identical to mkb_occupancy_grid_batch on that matrix. */
int mkb_occupancy_grid_batch_masked(mkb_handle_t h, void *stream, const float *coords, const double *radii,
                                    const uint32_t *chanmask, int64_t n_atoms, int32_t C, const mkb_grid_desc *grids,
                                    int32_t B, float *out, uint32_t flags);

/* K1 with a COMPACT result (end-to-end transfers): ~70 % of a pocket grid is empty, so instead of the dense grid the
 * kernel emits one 4 KB record [4 x][4 y][8 z][8 channels] per 4x4x8-voxel block that has an atom within 5 A, and an
 * index that says which blocks those are.  8 channels, voxel-major.  Block b of grid g (b = ((ix/4)*ceil(ny/4) +
 * iy/4)*ceil(nz/8) + iz/8, grids in batch order) has a record iff blk_rank[b + 1] != blk_rank[b]; the record is
 * records[1024 * blk_rank[b] ...].  records: device, room for mkb_occupancy_compact_blocks(grids, B) records in the
 * worst case; blk_rank: device uint32 [rank_capacity >= blocks + 1].  Exactly one of sigmas / (radii, chanmask) is given.
 * mkb_occupancy_expand_host rebuilds grids [g0, g1) of the dense float32 (sum M, 8) HOST array from host copies of the
 * records (`records` points at record rec0; NULL = only zero-fill the blocks without a record) with n_threads threads;
 * missing blocks are zero-filled; out_f64 != 0 writes
 * float64 (the reference's result dtype).  The result is bit-identical to mkb_occupancy_grid_batch. */
int mkb_occupancy_grid_batch_compact(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                                     const double *radii, const uint32_t *chanmask, int64_t n_atoms,
                                     const mkb_grid_desc *grids, int32_t B, float *records, uint32_t *blk_rank,
                                     int64_t rank_capacity);
int64_t mkb_occupancy_compact_blocks(const mkb_grid_desc *grids, int32_t B);
/* K1 straight into the caller's HOST array (end-to-end callers with a page-locked result, e.g. cudaHostAlloc / torch
 * pin_memory: under UVA such memory is device-accessible at the same address).  `out_mapped` is that dense float32
 * (sum M, 8) host array: the kernel stores the blocks that have an atom within 5 A directly into it over PCIe (TMA bulk
 * row copies, ~30 % of the bytes) and does not touch the others; the block index (as for the compact call) is computed before
 * the fill kernel starts and copied to `host_rank` (page-locked, blocks + 1 words) on a side stream, so the host can
 * zero-fill the empty blocks (mkb_occupancy_expand_host with records == NULL) WHILE the GPU computes and writes.
 * mkb_occupancy_wait_index blocks until host_rank has arrived; the caller synchronises `stream` before reading `out`. */
int mkb_occupancy_grid_batch_to_host(mkb_handle_t h, void *stream, const float *coords, const double *sigmas,
                                     const double *radii, const uint32_t *chanmask, int64_t n_atoms,
                                     const mkb_grid_desc *grids, int32_t B, float *out_mapped, uint32_t *blk_rank,
                                     int64_t rank_capacity, uint32_t *host_rank);
int mkb_occupancy_wait_index(mkb_handle_t h);
int mkb_occupancy_expand_host(const mkb_grid_desc *grids, int32_t g0, int32_t g1, const uint32_t *blk_rank,
                              const float *records, int64_t rec0, void *out, int32_t out_f64, int32_t n_threads);

/* Voxel centres on the device (SURVEY 8f row 1), exactly getCenters (voxeldescriptors.py:116-123,243-247):
 * centers[(out_offset_b + v) * 3 + d] = fl(fl(i_d * voxelsize) + origin[d]), v = (ix*ny + iy)*nz + iz; float64 device.
 * K1 itself never needs this array. */
int mkb_grid_centers(mkb_handle_t h, void *stream, const mkb_grid_desc *grids, int32_t B, double *centers);

/* rotateCoordinates (voxeldescriptors.py:78-114), batched (SURVEY 8f row 1): molecule b = atoms [atom_offsets[b],
 * atom_offsets[b+1]) (int64 device, [B+1]) is rotated three times in succession, new = (x - c_b) . R_{b,r}^T + c_b in
 * float64 (row-major 3x3 matrices [B][3][3][3] and centres [B][3], float64 device; the host wrapper builds the matrices
 * with the reference's rotationMatrix formula, util.py:101-117).  Result as float32 (what K1 consumes) and/or float64
 * (what the reference returns); either output may be NULL.  Products and sums individually rounded, left to right
 * (numpy's BLAS order is unspecified: parity is 1e-12 relative, not bitwise). */
int mkb_rotate_coords(mkb_handle_t h, void *stream, const float *coords, int64_t n_atoms, const int64_t *atom_offsets,
                      int32_t B, const double *matrices, const double *centers, float *out_f32, double *out_f64);

/* K1b: occupancy at arbitrary centres (the `usercenters` branch, voxeldescriptors.py:338-340 ->
 * calculate_occupancy).  centers [M,3] float64 device; same arithmetic contract. */
int mkb_occupancy_points(mkb_handle_t h, void *stream, const double *centers, int64_t M,
                         const float *coords, const double *sigmas, int64_t n_atoms, int32_t C,
                         float *out, uint32_t flags);

/* Trajectory view shared by the distance entry points: coords is float32 (n_atoms, 3, F) frame-minor
 * (moleculekit/molecule.py:144-146); element (a, d, f) lives at coords[(a*3 + d)*frame_stride + f], box (3, F) at
 * box[d*frame_stride_box + f].  A frame shard [f0, f1) of a resident trajectory is (coords + f0, n_frames = f1 - f0,
 * frame_stride = F). */
typedef struct {
    const float *coords;
    const float *box;
    int64_t n_atoms;
    int64_t n_frames;
    int64_t frame_stride;     /* elements between consecutive (atom, dim) rows of coords */
    int64_t frame_stride_box; /* elements between consecutive rows of box */
} mkb_traj;

/* K3: dist_trajectory (distance_utils.pyx:126-155) with the truncate / contacts post-ops of
 * pp_calcDistances (projections/util.py:74-84) fused into the store.
 *   sel1 [n1], sel2 [n2], chains [n_atoms] uint32 device; out [n_frames, P] row-major, P = n1*n2 or n1*(n1-1)/2
 *   when selfdist (then sel2 must equal sel1 as in the reference); float32 (mode 0) or uint8 (mode 1).
 *   truncate: NaN = off.  Arithmetic: every float op individually rounded (no FMA), roundf half-away, sqrtf IEEE
 *   -> bit-identical to the reference binary. */
int mkb_dist_trajectory(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                        const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist, int32_t pbc,
                        int32_t mode, float truncate, float threshold, void *out);

/* K4: contacts_trajectory (distance_utils.pyx:59-93), two calls.
 * count: row_offsets [n_frames*n1 + 1] int64 device receives the exclusive scan of the per-(frame, i) contact
 *        counts; *total_pairs (HOST) receives the grand total (this call synchronises the stream).
 * fill : pairs [total_pairs, 2] uint32 device receives (sel1[i], sel2[j]) in the reference's order: frame-major,
 *        then i ascending, then j ascending -- bit-exact index output.  thr2 = threshold*threshold in float
 *        (pyx:77), compare `<=`.
 * The count call keeps one hit mask per (row, 32 columns) in the handle; a fill call with the SAME arguments (pointers,
 * sizes, flags, threshold) emits the pairs from those masks instead of evaluating the distances again, any other fill call
 * recomputes them.  Either way the pairs are consistent with the row_offsets of the count call. */
int mkb_contacts_count(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                       const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist, int32_t pbc,
                       float threshold, int64_t *row_offsets, int64_t *total_pairs);
int mkb_contacts_fill(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                      const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist, int32_t pbc,
                      float threshold, const int64_t *row_offsets, uint32_t *pairs);

/* K5: dist_trajectory_reduction / dist_trajectory_reduction_pairs (distance_utils.pyx:211-350) with the same
 * fused post-ops (projections/util.py:212-223).  Groups are CSR (offsets [G+1] int64, atoms int32), device.
 * gchains1/2 [G1]/[G2] uint32 = chain id of each group's first atom (projections/util.py:174-179).
 * red1/red2: 0 closest, 1 centre of mass (float accumulation in atom order, pyx:160-183).
 * pairs != 0: group g of set 1 against group g of set 2 (G1 == G2), out [n_frames, G1];
 * else out [n_frames, G1*G2] or [n_frames, G1*(G1-1)/2] when selfdist. */
int mkb_dist_reduction(mkb_handle_t h, void *stream, const mkb_traj *t, const int64_t *g1_off,
                       const int32_t *g1_atoms, int64_t G1, const int64_t *g2_off, const int32_t *g2_atoms,
                       int64_t G2, const uint32_t *gchains1, const uint32_t *gchains2, int32_t selfdist,
                       int32_t pbc, const float *masses, int32_t red1, int32_t red2, int32_t pairs, int32_t mode,
                       float truncate, float threshold, void *out);

/* K6: cdist / pdist / squareform / get_collisions (distance_utils.pyx:355-435, 98-121).  Row-major float32. */
int mkb_cdist(mkb_handle_t h, void *stream, const float *a, int64_t n1, const float *b, int64_t n2, int32_t D,
              float *out);
int mkb_pdist(mkb_handle_t h, void *stream, const float *a, int64_t n, int32_t D, float *out);
int mkb_squareform(mkb_handle_t h, void *stream, const float *d, int64_t n, int64_t dim, float *out);
/* get_collisions: single frame, no pbc, LOCAL (i, j) indices; same two-call protocol as K4 with
 * row_offsets [n1 + 1]. */
int mkb_collisions_count(mkb_handle_t h, void *stream, const float *c1, int64_t n1, const float *c2, int64_t n2,
                         float threshold, int64_t *row_offsets, int64_t *total_pairs);
int mkb_collisions_fill(mkb_handle_t h, void *stream, const float *c1, int64_t n1, const float *c2, int64_t n2,
                        float threshold, const int64_t *row_offsets, uint32_t *pairs);

/* K8 (SURVEY 8f row 2): MetricShell radial histogram fused on the distance evaluation; replaces _shells
 * (moleculekit/projections/metricshell.py:183-202) and the (F, P) matrix it consumed.  counts [n_frames, n1, numshells]
 * uint32: partners j of centre sel1[c] with edges[e] < d <= edges[e+1] (edges [numshells+1] float64 device; d = the
 * reference's float32 distance, truncated if truncate is not NaN, compared in float64).  selfdist: sel2 == sel1 and a
 * centre is not its own partner.  1 <= numshells <= 32. */
int mkb_shell_counts(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                     const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist, int32_t pbc,
                     float truncate, const double *edges, int32_t numshells, uint32_t *counts);

/* K7 (stretch row a13): bond perception, replaces bond_grid_search (moleculekit/bondguesser.py:259-392) +
 * grid_bonds/_is_close (moleculekit/bondguesser_utils/bondguesser_utils.pyx:89-163).  coords [n,3] / radii [n] float32,
 * is_hydrogen [n] uint32, device.  pairdist = final grid box edge (after the caller's max_boxes enlargement loop).
 * Same two-call protocol as K4 with row_offsets [n + 1]; pairs come out as (i < j), unordered inside a row -- the SET
 * equals the reference's (the host wrapper returns it in canonical sorted order): pairs that pass _is_close AND lie in
 * the same or adjacent boxes floor(fl32(fl32(x - xyzmin) / pairdist)) of the reference's grid on every axis, xyzmin
 * being the per-axis minimum of coords (computed on the device). */
int mkb_bonds_count(mkb_handle_t h, void *stream, const float *coords, const float *radii, const uint32_t *is_hydrogen,
                    int64_t n, float pairdist, int64_t *row_offsets, int64_t *total_pairs);
int mkb_bonds_fill(mkb_handle_t h, void *stream, const float *coords, const float *radii, const uint32_t *is_hydrogen,
                   int64_t n, float pairdist, const int64_t *row_offsets, uint32_t *pairs);

/* K11 (SURVEY 8f row 4, second half): XTC compressed coordinates decoded on the device; replaces the frame loop of
 * xtc_read_new / xtc_read_frame (moleculekit/fileformats/xtc/src/xtc_src.cpp:195-258) around xdrfile_decompress_coord_float
 * (src/xdrfile.cpp:750-982) and its host-side scatter into the frame-minor array.  file_bytes = the XTC file on the device;
 * frames[f] (HOST) = one coordinate block as found by walking the XDR frame headers: byte offset and length of the bit stream,
 * precision, minint/maxint, initial smallidx (smallidx < 0: natoms <= 9, the block is 3*natoms big-endian floats).
 * coords (natoms, 3, n_frames) float32 device, element (a, d, f) at coords[(a*3 + d)*frame_stride + f], in nm, or multiplied
 * by `scale` as a second float32 operation (10 = the reference's `coords *= 10`, readers.py:1846).  status [n_frames] int32
 * device: 0 = ok, negative = corrupt block.  Blocks are read as big-endian 32-bit words: file_bytes + data_offset must be
 * 4-byte aligned (XDR guarantees it for a buffer that starts on a word) and readable up to the next multiple of 4 bytes.
 * Bit-identical to the reference reader. */
typedef struct {
    int64_t data_offset;
    int32_t nbytes;
    int32_t natoms;
    float precision;
    int32_t minint[3];
    int32_t maxint[3];
    int32_t smallidx;
} mkb_xtc_frame;
int mkb_xtc_decode(mkb_handle_t h, void *stream, const uint8_t *file_bytes, int64_t file_size, const mkb_xtc_frame *frames,
                   int64_t n_frames, int64_t natoms, float *coords, int64_t frame_stride, float scale, int32_t *status);

/* K21: XTC compressed coordinates written on the device, the inverse of K11; replaces xdrfile_compress_coord_float
 * (src/xdrfile.cpp) inside the frame loop of the reference's write_xtc.  coords float32 device, element (a, d, f) at
 * coords[(a*3 + d)*frame_stride + f]; every value is first multiplied by `scale` as a float32 operation of its own (1 = the
 * input is in nm, 0.1 = Angstrom in; skipped when scale == 1), then taken to the lattice at `precision` (<= 0 or NaN means
 * 1000) with the reference's individually rounded float32 steps.  Frame f's coordinate block -- what follows the second
 * atom count of its frame header in the file -- is written at out_bytes + frame_offsets[f], frame_nbytes[f] bytes long:
 *     natoms > 9:   precision (float), minint[3], maxint[3], smallidx, byte count of the bit stream (all 32-bit big-endian),
 *                   then the bit stream zero-padded to a multiple of 4 bytes
 *     natoms <= 9:  3*natoms big-endian floats
 * Blocks are packed back to back in frame order; every length is a multiple of 4 and out_bytes must be 4-byte aligned.
 * frame_offsets [n_frames + 1] int64, frame_nbytes [n_frames] int32 and status [n_frames] int32 are device arrays;
 * frame_offsets[n_frames] is the total.  A frame whose status is not 0 takes no bytes:
 *     MKB_XTC_ENC_COORD_OVERFLOW   a lattice coordinate beyond INT_MAX - 2 (or a coordinate that is not a number)
 *     MKB_XTC_ENC_RANGE_OVERFLOW   the lattice range of an axis reaches INT_MAX - 2
 *     (both are the reference's "Internal overflow compressing coordinates")
 *     MKB_XTC_ENC_SMALLIDX_RANGE   consecutive atoms so far apart that the reference would read past its table of ranges
 * The lengths are known only after a first pass over the frames, so this call synchronises the stream once (as
 * mkb_contacts_count does).  When the blocks need more than out_capacity bytes nothing is written to out_bytes and the
 * call returns MKB_ERR_CAPACITY with the three tables filled: frame_offsets[n_frames] is the capacity to come back with
 * (out_bytes may be NULL when out_capacity is 0).  n_frames == 0 or natoms == 0 returns MKB_OK and touches nothing.
 * Byte-identical to the reference writer. */
#define MKB_XTC_ENC_COORD_OVERFLOW (-1)
#define MKB_XTC_ENC_RANGE_OVERFLOW (-2)
#define MKB_XTC_ENC_SMALLIDX_RANGE (-3)
int mkb_xtc_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames, int64_t natoms,
                   float precision, float scale, uint8_t *out_bytes, int64_t out_capacity, int64_t *frame_offsets,
                   int32_t *frame_nbytes, int32_t *status);

/* K22: DCD (CHARMM / NAMD / OpenMM) frame records read on the device; replaces the per-frame fread and X/Y/Z -> xyz
 * interleave of read_charmm_timestep (moleculekit/fileformats/dcd/src/dcdplugin.c) and the host transposition to the
 * frame-minor array.  bytes = frame records on the device (4-byte aligned; every float of a DCD file sits at a multiple
 * of 4, since all its records and markers do); frames[k] (HOST) = listed frame k: the byte offsets in `bytes` of its X, Y
 * and Z float arrays and the floats per record.  coords (natoms, 3, n_frames) float32 device, element (a, d, k) at
 * coords[(a*3 + d)*frame_stride + k] = float a of record d of frame k.  Values are moved as 32-bit words, never through
 * float arithmetic: every bit pattern arrives unchanged.  swap != 0 byte-swaps every word (a file of the other byte order).
 * Fixed atoms (header NAMNF > 0): the file's first frame holds all natoms, every later frame only the n_free free atoms.
 * slot [natoms] int32 device = position of atom a in the free list, -1 for a fixed atom (NULL: no fixed atoms); a record
 * of natoms floats is indexed by atom, one of n_free floats by slot[a], and a fixed atom of such a frame is read from the
 * file's first frame, described by `first` (HOST) with offsets into first_bytes (device, first_nbytes long) -- so the first
 * frame is the source for fixed atoms even when it is not listed.  slot values must be below n_free.  Every descriptor is
 * checked on the host: a record outside its buffer, off a 4-byte boundary, or of another length is MKB_ERR_BAD_ARG.
 * Bit-identical to the plugin's reader. */
typedef struct {
    int64_t offset[3]; /* X, Y, Z float arrays */
    int64_t count;     /* floats per record: natoms, or n_free for a later frame of a file with fixed atoms */
} mkb_dcd_frame;
int mkb_dcd_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, const mkb_dcd_frame *frames,
                   int64_t n_frames, int64_t natoms, const int32_t *slot, int64_t n_free, const uint8_t *first_bytes,
                   int64_t first_nbytes, const mkb_dcd_frame *first, int32_t swap, float *coords, int64_t frame_stride);

/* K22: DCD frame records written on the device, the inverse of mkb_dcd_decode; replaces the frame loop of the plugin's
 * write_dcdstep.  coords float32 device, element (a, d, k) at coords[(a*3 + d)*frame_stride + k]; unitcell [n_frames][6]
 * float64 device (A, cos gamma, B, cos beta, cos alpha, C) or NULL.  Frame k is written at out + k*S, S = 56 (with a unit
 * cell) + 3*(8 + 4*natoms) bytes: the unit-cell record [48, 6 doubles, 48] when unitcell != NULL, then the X, Y and Z
 * records [4*natoms, natoms floats, 4*natoms], all little-endian (the plugin's native order on x86), no fixed atoms.  out
 * is 4-byte aligned, unitcell 8-byte aligned; n_frames*S > out_capacity is MKB_ERR_CAPACITY and 4*natoms beyond the
 * int32 record markers MKB_ERR_BAD_ARG.  Byte-identical to the plugin's frame records. */
int mkb_dcd_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames, int64_t natoms,
                   const double *unitcell, uint8_t *out, int64_t out_capacity);

/* K23: AMBER NetCDF (netCDF-3) trajectory coordinates read on the device; replaces the host read of the big-endian
 * `coordinates` variable (frame, atom, spatial) (moleculekit/fileformats/netcdf.py) and the host transposition to the
 * frame-minor array.  bytes = staged file bytes on the device (4-byte aligned); offsets[k] (HOST) = byte offset in
 * `bytes` of listed frame k's 12*natoms coordinate bytes (big-endian float32, atom-major, x y z per atom), >= 0, a
 * multiple of 4 and with offsets[k] + 12*natoms <= nbytes, else MKB_ERR_BAD_ARG.  coords (natoms, 3, n_frames) float32
 * device, element (a, d, k) at coords[(a*3 + d)*frame_stride + k].  Values are byte-swapped as 32-bit words, never
 * passed through float arithmetic: every bit pattern arrives unchanged. */
int mkb_netcdf_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, const int64_t *offsets,
                      int64_t n_frames, int64_t natoms, float *coords, int64_t frame_stride);

/* K23: AMBER NetCDF records written on the device, the inverse of mkb_netcdf_decode.  coords float32 device, element
 * (a, d, k) at coords[(a*3 + d)*frame_stride + k].  Record k is written at out + k*record_bytes: its coordinates
 * big-endian at coord_offset, and the other record_bytes - 12*natoms bytes from extra + k*(record_bytes - 12*natoms)
 * (device, already in file byte order; NULL when there are none): the first coord_offset of them before the
 * coordinates, the rest after.  record_bytes and coord_offset are multiples of 4 with coord_offset + 12*natoms <=
 * record_bytes; out, extra and coords are 4-byte aligned.  n_frames*record_bytes > out_capacity is MKB_ERR_CAPACITY. */
int mkb_netcdf_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                      int64_t natoms, int64_t record_bytes, int64_t coord_offset, const uint8_t *extra, uint8_t *out,
                      int64_t out_capacity);

/* K24: GROMACS TRR x, v or f blocks read on the device; replaces xdrfile's read_trr (moleculekit/fileformats/xtc/trr.pyx
 * over xdrfile_trr.c), which returns each frame's block as (natoms, 3) reals, and the host transposition to the
 * frame-minor array.  bytes = staged file bytes on the device; offsets[k] (HOST) = byte offset in `bytes` of listed frame
 * k's block: 3*natoms big-endian XDR reals of value_bytes (4: float32, 8: float64) each, atom-major, x y z per atom.
 * value_bytes is 4 or 8; bytes and every offset are multiples of value_bytes, offsets[k] >= 0 and offsets[k] +
 * 3*natoms*value_bytes <= nbytes, else MKB_ERR_BAD_ARG.  A float64 block in a file starts on a 4-byte boundary only (the
 * double-precision header is 92 bytes), so 8-byte reals are read with 64-bit loads from a staging buffer the caller
 * lays out at multiples of 8 (moleculekit_b200.trr stages every block in its own row of 24*natoms bytes), not from the
 * file's own offsets.  coords (natoms, 3, n_frames) float32 device, element (a, d, k) at coords[(a*3 + d)*frame_stride +
 * k].  4-byte reals are byte-swapped as 32-bit words, never passed through float arithmetic: every bit pattern arrives
 * unchanged.  8-byte reals are rounded to float32 exactly as x86-64's cvtsd2ss (numpy's astype(np.float32)) does:
 * to nearest, ties to even, overflow to +-inf, float32 subnormals kept; a NaN gives sign | 0x7fc00000 | (its 52-bit
 * mantissa >> 29). */
int mkb_trr_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, const int64_t *offsets,
                   int64_t n_frames, int64_t natoms, int32_t value_bytes, float *coords, int64_t frame_stride);

/* K24: single-precision GROMACS TRR frames written on the device, the inverse of mkb_trr_decode for 4-byte reals;
 * replaces the frame loop of xdrfile's write_trr.  x, v, f float32 device (v and f NULL when absent), each element
 * (a, d, k) at p[(a*3 + d)*frame_stride + k]: one frame stride for all three.  Frame k is written at out + k*R, R =
 * head_bytes + (1 + (v != NULL) + (f != NULL))*12*natoms: its head_bytes bytes from head + k*head_bytes (device, already
 * in file byte order -- the writer puts the 84-byte frame header and the 36-byte box there), then x, then v and f when
 * given, each as 3*natoms big-endian float32.  head_bytes is a multiple of 4; x, v, f, head and out are 4-byte aligned.
 * n_frames*R > out_capacity is MKB_ERR_CAPACITY.  Values are byte-swapped as 32-bit words: every bit pattern is
 * written unchanged. */
int mkb_trr_encode(mkb_handle_t h, void *stream, const float *x, const float *v, const float *f, int64_t frame_stride,
                   int64_t n_frames, int64_t natoms, const uint8_t *head, int64_t head_bytes, uint8_t *out,
                   int64_t out_capacity);

/* K25: AMBER ASCII trajectory (mdcrd / mdvel) frames parsed on the device; replaces a host reader that converts every
 * 8-character field with float() and the host transposition to the frame-minor array.  A frame holds 3*natoms F8.3
 * fields atom-major (x y z per atom), ten to a line: value j at byte 8*j + j/10, a newline after every value with
 * j % 10 == 9 and after the last; with with_box != 0 one more line of three F8.3 fields (A, B, C) and a newline.  Frame
 * bytes S = 24*natoms + ceil(3*natoms/10) + (with_box ? 25 : 0).  A field is spaces, an optional '-', digits, '.' and
 * three digits.  bytes = staged file bytes on the device, 16-byte aligned; offsets[k] (HOST) = byte offset in `bytes`
 * of listed frame k, >= 0, a multiple of 16, with offsets[k] + S rounded up to 4 <= nbytes (the kernel reads whole
 * aligned words), else MKB_ERR_BAD_ARG.  coords (natoms, 3, n_frames) float32 device, element (a, d, k) at
 * coords[(a*3 + d)*frame_stride + k]; box (3, n_frames) float32 device at box[d*box_stride + k], used only with a box.
 * A field's digits k (point removed) give __double2float_rn(k / 1000.0) with its sign, bit for bit
 * np.float32(float(field)) ('-0.000' is -0.0).  bad (device int64, 8-byte aligned, set to INT64_MAX by the caller)
 * receives the atomic minimum of k*S + b over the malformed bytes b of listed frame k: a field that breaks the grammar
 * (b = its first byte) or a byte that is not the newline the layout puts there.  The values decoded from a malformed
 * frame are unspecified. */
int mkb_mdcrd_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, const int64_t *offsets,
                     int64_t n_frames, int64_t natoms, int32_t with_box, float *coords, int64_t frame_stride,
                     float *box, int64_t box_stride, int64_t *bad);

/* K25: AMBER ASCII trajectory frames written on the device, the inverse of mkb_mdcrd_decode.  coords float32 device,
 * element (a, d, k) at coords[(a*3 + d)*frame_stride + k]; box (3, n_frames) float32 device at box[d*box_stride + k], or
 * NULL for frames without a box line.  Frame k is written at out + k*S (S as for mkb_mdcrd_decode, with_box = box !=
 * NULL), byte for byte Python's '%8.3f' % x: k = rint(x * 1000) in float64 (exact, half to even), the sign printed
 * whenever x is negative or -0.0.  A value outside the writable range (rint(x * 1000) > 9 999 999 for x >= 0, < -999 999
 * for x < 0) or not finite is written as '********'.  The title line is the caller's.  coords, box and out are 4-byte
 * aligned; n_frames*S > out_capacity is MKB_ERR_CAPACITY. */
int mkb_mdcrd_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                     int64_t natoms, const float *box, int64_t box_stride, uint8_t *out, int64_t out_capacity);

/* K26: the index pass over a chunk of a multi-frame XYZ file; replaces the host reader's line loop (readline, split()
 * and int() per frame) as far as finding the frames.  A frame is P = natoms + 2 lines: the atom count, a comment and
 * natoms atom lines.  bytes = the chunk on the device, 16-byte aligned: the file's bytes [file_base, file_base + n_read),
 * of which the newlines in the first n are counted (n_read - n bytes of look-ahead, up to 64, let the last lines of the
 * chunk be checked).  state (device int64[3], 8-byte aligned; the caller sets {0, INT64_MAX, 0} before the first chunk
 * and keeps it across chunks, which run in file order on one stream): [0] the running newline count, [1] the atomic
 * minimum file offset of a CR not followed by LF, [2] one more than the largest frame number past frame_cap.  Every line
 * L (0-based in the file) with L % P == 0 and L >= P that starts inside the look-ahead window gets frame_off[L / P] =
 * its file offset and status[L / P] = 0 when its first field is natoms written as [+]digits (ASCII separators before
 * it, a separator after it, within 64 bytes), 1 when the host must decide (frame_off, status device, frame_cap
 * entries).  Frame 0 is the caller's. */
int mkb_xyz_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read, int64_t file_base,
                  int64_t natoms, int64_t *state, int64_t *frame_off, uint8_t *status, int64_t frame_cap);

/* K26: XYZ frames parsed on the device; replaces the host reader's split() and float() per atom line and the host
 * transposition to the frame-minor array.  bytes = n_staged whole frames back to back on the device, 16-byte aligned,
 * nbytes long and readable up to nbytes rounded up to 16; each frame's P = natoms + 2 lines end in '\n' (the last
 * frame's last line may end at nbytes instead).  frame_of (HOST int32[n_frames]) = the staged frame of listed frame k.
 * coords (natoms, 3, n_frames) float32 device, element (a, d, k) at coords[(a*3 + d)*frame_stride + k] = field d + 1 of
 * atom line a, bit for bit np.float32(float(field)): the correctly rounded double rounded to float32 (field 0 and
 * fields past 3 are skipped).  Separators are the bytes str.split() splits ASCII text on (\t \n \v \f \r, space,
 * 0x1c-0x1f).  A line with fewer than four fields, a byte >= 0x80 up to its fourth field, a field outside
 * [+-]?(d+.?d*|.d+)([eE][+-]?d+)? and nan / inf / infinity, or a conversion the device cannot decide is flagged: flags
 * (device int64, 8-byte aligned, flags[0] set to 0 by the caller) receives at flags[1 + 2 j], flags[2 + 2 j] the pair
 * ((frame_base + k) * natoms + a, byte offset of the line from its frame's first byte) for j < flag_cap, and flags[0]
 * counts every flagged line; such a line's coordinates are unspecified. */
int mkb_xyz_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                   const int32_t *frame_of, int64_t n_frames, int64_t natoms, float *coords, int64_t frame_stride,
                   int64_t frame_base, int64_t *flags, int64_t flag_cap);

/* K26: XYZ frames written on the device, the inverse of mkb_xyz_decode.  coords float32 device, element (a, d, k) at
 * coords[(a*3 + d)*frame_stride + k].  Frame k is written at out + k*S, S = head_bytes + natoms*(width + 49): the
 * head_bytes bytes of head (device: the count and comment lines), then per atom its element column elements[a*width
 * ...] (device, width bytes, 1 <= width <= 256) and ' %15.8f' of x, y and z, and '\n': byte for byte Python's
 * '%-*s %15.8f %15.8f %15.8f\n'.  k = rint(x * 1e8) in float64 (exact, half to even); the caller keeps |k| below 10^14
 * (10^13 for a negative sign) and NaN / inf out.  coords and out are 4-byte aligned; n_frames*S > out_capacity is
 * MKB_ERR_CAPACITY. */
int mkb_xyz_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                   int64_t natoms, const uint8_t *head, int64_t head_bytes, const uint8_t *elements, int64_t width,
                   uint8_t *out, int64_t out_capacity);

/* K28: the index pass over a chunk of a multi-model PDB file; replaces the host reader's line loop as far as finding
 * the frames.  The frame rules (the host applies them to the list this pass builds):
 *   - an atom record is a line whose first six bytes are "ATOM  " or "HETATM"; every other record is skipped;
 *   - with MODEL records (first five bytes "MODEL", then a space or the line's end) each MODEL starts a frame that runs
 *     to the next MODEL, ENDMDL or END record (first three bytes "END", then a space or the line's end) or the end of
 *     the file; without them the file is one frame of the atom records before the first ENDMDL / END;
 *   - natoms is frame 0's atom record count and every other frame holds exactly natoms; a last model cut short by the
 *     end of the file (no ENDMDL / END after it) is dropped;
 *   - a frame's cell is the last CRYST1 record before its first atom record.
 * bytes = the chunk on the device, 16-byte aligned: the file's bytes [file_base, file_base + n_read), of which the line
 * starts after the newlines in the first n are classified (n_read - n bytes of look-ahead, at least 6, let the last
 * lines be read); byte 0 starts a line when file_base == 0.  state (device int64[3], 8-byte aligned; the caller sets
 * {0, INT64_MAX, 0} before the first chunk and keeps it across chunks, which run in file order on one stream): [0] the
 * running atom record count, [1] the atomic minimum file offset of a CR not followed by LF, [2] the number of marks.
 * Every MODEL, ENDMDL, END and CRYST1 record appends (file offset * 8 + kind, atom records before it in the file) to
 * marks (device int64[2 * mark_cap]) at slot state[2]++ while the slot is below mark_cap; kind 2 MODEL, 3 ENDMDL, 4 END,
 * 5 CRYST1.  The slots are in no particular order. */
int mkb_pdb_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read, int64_t file_base,
                  int64_t *state, int64_t *marks, int64_t mark_cap);

/* K28: PDB frames parsed on the device; replaces the host reader's float() of columns 31-38, 39-46 and 47-54 of every
 * atom record and the host transposition to the frame-minor array.  bytes = n_staged whole frames back to back on the
 * device, 16-byte aligned, nbytes long and readable up to nbytes rounded up to 16; each staged frame starts a line,
 * holds exactly natoms atom records and (but for the last) ends in '\n'.  frame_of (HOST int32[n_frames]) = the staged
 * frame of listed frame k.  coords (natoms, 3, n_frames) float32 device, element (a, d, k) at coords[(a*3 + d)*
 * frame_stride + k] = field d of atom record a, bit for bit np.float32(float(field)): the F8.3 fast path, else the
 * grammar of mkb_xyz_decode within the 8-byte field.  A line shorter than 54 columns (a '\n' or '\r' before column 55),
 * an empty field, a field outside the grammar, a byte >= 0x80 or an undecided rounding is flagged: flags (device int64,
 * 8-byte aligned, flags[0] set to 0 by the caller) receives (frame_base + k) * natoms + a at flags[1 + j] for j <
 * flag_cap, and flags[0] counts every flagged line; such a line's coordinates are unspecified. */
int mkb_pdb_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                   const int32_t *frame_of, int64_t n_frames, int64_t natoms, float *coords, int64_t frame_stride,
                   int64_t frame_base, int64_t *flags, int64_t flag_cap);

/* K28: CRYST1 records parsed on the device.  rows (device, 16-byte aligned) holds n_cells rows of 64 bytes, each the
 * first 54 (or more) bytes of a CRYST1 line.  cells (device float32[6 * n_cells]) = a, b, c (columns 7-15, 16-24,
 * 25-33) and alpha, beta, gamma (columns 34-40, 41-47, 48-54) of row i at cells[6 i + d], each bit for bit
 * np.float32(float(field)); bad (device int32[n_cells]) = 1 where the row's fields are left to the host (as for
 * mkb_pdb_decode's flags), else 0. */
int mkb_pdb_cell(mkb_handle_t h, void *stream, const uint8_t *rows, int64_t n_cells, float *cells, int32_t *bad);

/* K28: PDB frames written on the device, the inverse of mkb_pdb_decode.  coords float32 device, element (a, d, k) at
 * coords[(a*3 + d)*frame_stride + k]; box and angles (3, n_frames) float32 device at [d*box_stride + k], or box NULL for
 * frames without a CRYST1 line.  Frame k is written at out + k*S, S = 15 + (box ? 71 : 0) + 81*natoms + 7:
 * "MODEL %8d\n" of model0 + k + 1, with a box "CRYST1%9.3f%9.3f%9.3f%7.2f%7.2f%7.2f P 1           1\n", then per atom
 * the 81 bytes of tmpl[a*81 ...] (device, readable up to 81*natoms rounded up to 4) with '%8.3f' of x, y and z in
 * columns 31-54, then "ENDMDL\n".  Each field is byte for byte Python's '%W.Df': rint(x * 10^D) in float64 (exact,
 * half to even), the sign printed whenever x is negative or -0.0; the caller keeps every value inside its field and
 * model0 + n_frames <= 10^8.  coords, tmpl, box, angles and out are 4-byte aligned; n_frames*S > out_capacity is
 * MKB_ERR_CAPACITY. */
int mkb_pdb_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                   int64_t natoms, const uint8_t *tmpl, const float *box, const float *angles, int64_t box_stride,
                   int64_t model0, uint8_t *out, int64_t out_capacity);

/* K30: the index pass over a chunk of the _atom_site loop body of a PDBx/mmCIF file; replaces the host reader's
 * tokenizer as far as finding the frames.  The rules (the host applies them to what this pass returns):
 *   - a line whose first non-blank byte is '#' (a comment) or '\n' is skipped; the body ends at the first line whose first
 *     token is a tag ('_...'), loop_, stop_ or global_, or starts with data_ or save_ (letters in any case); every other
 *     line is a row;
 *   - blanks are space, \t, \v, \f and \r; a token is a run of other bytes, or a '...' / "..." string that opens at the
 *     token's start and closes at the first matching quote followed by a blank or the line's end;
 *   - a row holds exactly n_tags tokens, and its token model_col (when model_col >= 0) is an unquoted [+-]?digits of at
 *     most 18 digits; a row starting with ';' (a text field) or with a quote that does not close is bad;
 *   - a frame is a maximal run of rows with the same model number (model_col -1: the whole loop is one frame).
 * bytes = the chunk on the device, 16-byte aligned: the file's bytes [file_base, file_base + n_read), of which the line
 * starts after the newlines in the first n are classified (n_read - n bytes of look-ahead let the last rows be read
 * whole); byte 0 starts a line when first != 0.  state (device int64[7], 8-byte aligned; the caller sets {0, INT64_MAX,
 * 0, INT64_MAX, INT64_MAX, INT64_MIN, -1} before the first chunk and keeps it across chunks, which run in file order on
 * one stream): [0] the running row count, [1] the minimum file offset of a CR not followed by LF before the body's end,
 * [2] the number of marks, [3] the minimum file offset of a bad row, [4] the minimum file offset of a line that ends the
 * body, [5] the model number of the last row so far (INT64_MIN: none), [6] the rows before the body's end once that
 * line has been seen, else -1.  Every row before the body's end whose model number differs from the row before it
 * appends (file offset, rows before it, model number) to marks (device int64[3 * mark_cap]) at slot state[2]++ while
 * the slot is below mark_cap; the slots are in no particular order. */
int mkb_cif_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read, int64_t file_base,
                  int64_t first, int64_t n_tags, int64_t model_col, int64_t *state, int64_t *marks, int64_t mark_cap);

/* K30: mmCIF frames parsed on the device; replaces the host reader's tokenizer and float() of the Cartn_x, Cartn_y and
 * Cartn_z tokens of every row and the host transposition to the frame-minor array.  bytes = n_staged whole frames back
 * to back on the device, 16-byte aligned, nbytes long and readable up to nbytes rounded up to 16; each staged frame
 * starts a line, holds exactly natoms rows (comment and blank lines between them are skipped, as by mkb_cif_index) and
 * (but for the last) ends in '\n'.  frame_of (HOST int32[n_frames]) = the staged frame of listed frame k.  coords
 * (natoms, 3, n_frames) float32 device, element (a, d, k) at coords[(a*3 + d)*frame_stride + k] = token col_x, col_y or
 * col_z (0-based) of row a, bit for bit np.float32(float(token)) in the grammar of mkb_xyz_decode.  A quoted token, a
 * token outside the grammar ('?', '.', '1.5(2)', ...), a byte >= 0x80 before the last of the three tokens, a row with
 * fewer tokens or an undecided rounding is flagged as in mkb_pdb_decode: flags[1 + j] = (frame_base + k) * natoms + a for
 * j < flag_cap, flags[0] counts every flagged row; such a row's coordinates are unspecified. */
int mkb_cif_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                   const int32_t *frame_of, int64_t n_frames, int64_t natoms, int64_t col_x, int64_t col_y,
                   int64_t col_z, float *coords, int64_t frame_stride, int64_t frame_base, int64_t *flags,
                   int64_t flag_cap);

/* K30: mmCIF rows written on the device, the inverse of mkb_cif_decode.  coords float32 device, element (a, d, k) at
 * coords[(a*3 + d)*frame_stride + k].  Frame k is written at out + k*S, S = natoms*row_bytes: per atom the row_bytes of
 * tmpl[a*row_bytes ...] (device, readable up to natoms*row_bytes rounded up to 4; row_bytes <= 768) with id =
 * (frame0 + k)*natoms + a + 1 right-justified in id_width bytes at col_id, '%10.3f' of x, y and z at col_x, col_x + 11
 * and col_x + 22, and pdbx_PDB_model_num = frame0 + k + 1 right-justified in model_width bytes at col_model.  Each field
 * is byte for byte Python's '%10.3f' (as mkb_pdb_encode's fields); the caller keeps every value inside its field.  coords,
 * tmpl and out are 4-byte aligned; n_frames*S > out_capacity is MKB_ERR_CAPACITY. */
int mkb_cif_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                   int64_t natoms, const uint8_t *tmpl, int64_t row_bytes, int64_t col_id, int64_t id_width,
                   int64_t col_x, int64_t col_model, int64_t model_width, int64_t frame0, uint8_t *out,
                   int64_t out_capacity);

/* K31: one BinaryCIF column decoded on the device; replaces a host reader's per-value loops over the column's encodings.
 * data = the column's bytes on the device (16-byte aligned, nbytes long).  steps (HOST double[6 * n_steps]) = the
 * encodings in decode order (the reverse of the file's list), six words each, unused words 0:
 *   {1, type}                         ByteArray, first and only first: little-endian values, type Int8 1, Int16 2,
 *                                     Int32 3, Uint8 4, Uint16 5, Uint32 6 (to 32-bit integers), Float32 32 or Float64 33
 *                                     (to float32, rounded to nearest even); nbytes a multiple of the type's size;
 *   {2, byteCount, isUnsigned, srcSize}   IntegerPacking (byteCount 1 or 2): an element equal to a limit (0xFF / 0xFFFF
 *                                     unsigned, 0x7F or -0x80 / 0x7FFF or -0x8000 signed) is added to the next one;
 *   {3, origin, srcType}              Delta: out[0] = origin + d[0], out[i] = out[i-1] + d[i] modulo 2^width(srcType);
 *   {4, srcType, srcSize}             RunLength: (value, count) pairs, values narrowed to srcType;
 *   {5, factor, srcType}              FixedPoint, last: float32(double(q) / factor);
 *   {6, min, max, numSteps, srcType}  IntervalQuantization, last: float32(min + ((max - min) / (numSteps - 1)) * q), each
 *                                     float64 operation rounded on its own.
 * Integers wrap modulo 2^32; a Uint32 array keeps its values as unsigned.  Every array holds at most 2^31 - 2 values.
 * mode 0 (rows): out[i] = decoded value i for i < n_out (int32 or float32 bits, 4-byte words).  mode 1 (frames): the
 * column holds whole frames of natoms rows, floats; out[a*atom_stride + k] = value of row frames[k]*natoms + a for
 * frames (HOST int64[n_out], any order, repeats allowed) and atom_stride >= n_out (an axis of (natoms, 3, F) frame-minor
 * float32 coords: coords + axis*frame_stride with atom_stride = 3*frame_stride).  mode 2 (runs): integers; every row i
 * whose value differs from row i-1 (and row 0) appends (i, value) to out (device int64[2 * n_out]) at slot status[1]++
 * while the slot is below n_out, slots in no particular order.  status (device int64[2], 8-byte aligned, zeroed by the
 * call): [0] 0, or the first data error found: 1 an IntegerPacking that ends inside a value, 2 one that holds another
 * number of values than srcSize, 3 RunLength counts that do not sum to srcSize, 4 a negative count (the outputs are then
 * unspecified); [1] the runs of mode 2.  A chain that does not fit these rules is MKB_ERR_BAD_ARG.  out is 4-byte
 * aligned (mode 2: 8-byte).  Nothing is synchronised; the caller keeps data, out and status valid until the stream reaches the end. */
int mkb_bcif_decode(mkb_handle_t h, void *stream, const uint8_t *data, int64_t nbytes, const double *steps,
                    int64_t n_steps, int64_t mode, void *out, int64_t n_out, const int64_t *frames, int64_t natoms,
                    int64_t atom_stride, int64_t *status);

/* K31: q[k*natoms + a] = rint(double(x[a*atom_stride + k*frame_stride]) * factor) (half to even) for every atom a and
 * frame k: one axis of a frame-minor (natoms, 3, F) float32 array (x = coords + axis*frame_stride, atom_stride =
 * 3*frame_stride, frame stride 1) quantized in BinaryCIF's row order.  x and q (device int32[natoms * n_frames]) are
 * 4-byte aligned; the caller keeps every value finite with its quantum inside int32. */
int mkb_bcif_quantize(mkb_handle_t h, void *stream, const float *x, int64_t atom_stride, int64_t frame_stride,
                      int64_t natoms, int64_t n_frames, double factor, int32_t *q);

/* K31: the sizes of the BinaryCIF encoder's four chains of one int32 array, for the host to choose one.  The array has
 * n values (1 to 2^31 - 2), value i = v[i % period] + (i / period) * step modulo 2^32 (v device int32[period], 4-byte
 * aligned; step 0 and period n for a plain array).  Its deltas are d[0] = 0, d[i] = value i - value i-1 (modulo 2^32),
 * and a run-length array is the (value, count) pairs of its maximal runs.  sizes (HOST int64[25]): [0] value 0, then
 * for the chains (a) the array, (b) its run-length array, (c) its deltas, (d) their run-length array, six words each:
 * length, minimum, and the elements IntegerPacking takes at 1 byte unsigned, 2 bytes unsigned, 1 byte signed and 2 bytes
 * signed, each value v counting floor(|v| / |limit|) + 1 with the limit on v's side (unsigned sums count negative
 * values as 0).  Synchronises the stream. */
int mkb_bcif_sizes(mkb_handle_t h, void *stream, const int32_t *v, int64_t period, int64_t step, int64_t n,
                   int64_t *sizes);

/* K31: the payload of one chain of mkb_bcif_sizes's array (same v, period, step, n): chain 0 to 3 for (a) to (d) and
 * n_packed its length as mkb_bcif_sizes reported it.  width 4 writes the chain's array as little-endian int32 (ByteArray
 * Int32, 4 * n_packed bytes); width 1 or 2 writes it IntegerPacked (signed, or with is_unsigned unsigned: the caller
 * checked that no value is negative) as little-endian Int8 / Int16 / Uint8 / Uint16 elements, as many as
 * mkb_bcif_sizes counted.  out (device, 4-byte aligned) holds out_bytes; elements past it are not written, and width 4
 * with 4 * n_packed > out_bytes is MKB_ERR_CAPACITY.  Nothing is synchronised. */
int mkb_bcif_emit(mkb_handle_t h, void *stream, const int32_t *v, int64_t period, int64_t step, int64_t n, int64_t chain,
                  int64_t width, int64_t is_unsigned, int64_t n_packed, uint8_t *out, int64_t out_bytes);

/* K29: the index pass over a chunk of a multi-frame GROMACS GRO file; replaces the host reader's line loop as far as
 * finding the frames.  The format: a frame is P = natoms + 3 lines -- a title (free text, GROMACS writes "t= <time>
 * step= <step>" into it), the atom count (a free-format integer), natoms atom lines ("%5d%-5s%5s%5d": resid, resname,
 * atom name, serial, then three position fields of width w in nm and optionally three velocity fields of width w in
 * nm/ps) and a box line (free format: 3 values v1x v2y v3z or 9 values v1x v2y v3z v1y v1z v2x v2z v3x v3y, in nm).
 * bytes = the chunk on the device, 16-byte aligned: the file's bytes [file_base, file_base + n_read), of which the
 * newlines in the first n are counted (n_read - n bytes of look-ahead, up to 64, let the last count lines be checked).
 * state (device int64[3], 8-byte aligned; the caller sets {0, INT64_MAX, 0} before the first chunk and keeps it across
 * chunks, which run in file order on one stream): [0] the running newline count, [1] the atomic minimum file offset of
 * a CR not followed by LF, [2] one more than the largest frame number past frame_cap.  Line L (0-based in the file)
 * with L % P == 0 and L >= P that starts inside the look-ahead window gets frame_off[L / P] = its file offset; line L
 * with L % P == 1 gets status[L / P] = 0 when its first field is natoms written as [+]digits (ASCII separators before
 * it, a separator after it, within 64 bytes), 1 when the host must decide (frame_off, status device, frame_cap
 * entries). */
int mkb_gro_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read, int64_t file_base,
                  int64_t natoms, int64_t *state, int64_t *frame_off, uint8_t *status, int64_t frame_cap);

/* K29: GRO frames parsed on the device; replaces the host reader's column slices and float() per atom line and the host
 * transposition to the frame-minor arrays.  bytes = n_staged whole frames back to back on the device, 16-byte aligned,
 * nbytes long and readable up to nbytes rounded up to 16; each frame's P = natoms + 3 lines end in '\n' (the last
 * frame's last line may end at nbytes instead).  frame_of (HOST int32[n_frames]) = the staged frame of listed frame k.
 * Atom line a must hold cols = 20 + 3 width characters (20 + 6 width when `velocities`, the file's velocity flag)
 * before its '\n' or CRLF.  coords (natoms, 3, n_frames) float32 device, element (a, d, k) at coords[(a*3 + d)*
 * frame_stride + k] = the width-character field at column 20 + width d of atom line a, bit for bit
 * np.float32(float(field)); vels (NULL, or with `velocities` the same layout and stride) = the fields at column 20 +
 * width (3 + d).  For width 8 the F8.3 (positions) and F8.4 (velocities) fast paths run first, else and for the fields
 * they reject the grammar of mkb_xyz_decode within the field.  A short line, an empty field, a field outside the
 * grammar, a byte >= 0x80 or an undecided rounding is flagged: flags (device int64, 8-byte aligned, flags[0] set to 0
 * by the caller) receives (frame_base + k) * natoms + a at flags[1 + j] for j < flag_cap, and flags[0] counts every
 * flagged line; such a line's values are unspecified.  1 <= width <= 32. */
int mkb_gro_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                   const int32_t *frame_of, int64_t n_frames, int64_t natoms, int64_t width, int32_t velocities,
                   float *coords, float *vels, int64_t frame_stride, int64_t frame_base, int64_t *flags,
                   int64_t flag_cap);

/* K29: the title and box lines of staged GRO frames parsed on the device.  Staged frame u is bytes[frame_at[u],
 * frame_at[u + 1]) (bytes and frame_at device, frame_at int64[n_staged + 1]).  box (device float32[9 n_staged]): the
 * ASCII-whitespace-separated tokens of the frame's last line in file order at box[9 u + t], each bit for bit
 * np.float32(float(token)); time (device float64[n_staged]) = float() of the token after the first " t= " of the
 * frame's first line, NaN without one; step (device int64[n_staged]) = the integer after the first " step= ", -1
 * without one.  status (device int32[n_staged]): bit 0 when the box line does not hold 3 or 9 tokens or holds a token
 * the device does not decide, bit 1 when the time token, bit 2 when the step token is left to the host ([+-] and at
 * most 18 digits are decided); the values under a set bit are unspecified. */
int mkb_gro_head(mkb_handle_t h, void *stream, const uint8_t *bytes, const int64_t *frame_at, int64_t n_staged,
                 float *box, double *time, int64_t *step, int32_t *status);

/* K29: GRO frames written on the device, the inverse of mkb_gro_decode.  coords float32 device, element (a, d, k) at
 * coords[(a*3 + d)*frame_stride + k]; vels NULL or the same layout; box (3, 3, n_frames) float32 device, component j of
 * box vector i at box[(3 i + j)*box_stride + k].  Frame k is written at out + k*S, S = head_bytes + natoms*L + B, L =
 * 69 with vels else 45, B = 91 when box9 else 31: the head_bytes bytes head[k*head_bytes ...] (device: the frame's
 * title and count lines), then per atom its 20 bytes prefix[a*20 ...] (device), '%8.3f' of x, y, z, with vels '%8.4f'
 * of vx, vy, vz, and '\n'; then '%10.5f' of v1x v2y v3z (box9: and v1y v1z v2x v2z v3x v3y) and '\n'.  Each field is
 * byte for byte Python's '%W.Df': rint(x * 10^D) in float64 (exact, half to even), the sign printed whenever x is
 * negative or -0.0; the caller keeps every value inside its field.  coords, vels, prefix, box and out are 4-byte
 * aligned; n_frames*S > out_capacity is MKB_ERR_CAPACITY. */
int mkb_gro_encode(mkb_handle_t h, void *stream, const float *coords, const float *vels, int64_t frame_stride,
                   int64_t n_frames, int64_t natoms, const uint8_t *head, int64_t head_bytes, const uint8_t *prefix,
                   const float *box, int64_t box_stride, int32_t box9, uint8_t *out, int64_t out_capacity);

/* K32: the index pass over a chunk of a LAMMPS dump file (dump atom / dump custom text); replaces the host reader's
 * line loop as far as finding and checking the frames.  A frame is P = H + natoms lines: H header lines (ITEM: TIME and
 * its value, ITEM: TIMESTEP and its value, ITEM: NUMBER OF ATOMS and the count, ITEM: BOX BOUNDS and three bound lines,
 * ITEM: ATOMS and its column names, in frame 0's order) and natoms atom lines; frame 0 may start with an ITEM: UNITS
 * pair the later frames lack.  bytes = the chunk on the device, 16-byte aligned: the file's bytes [file_base, file_base
 * + n_read), of which the newlines in the first n are counted (the look-ahead lets a header that starts in the chunk
 * be checked).  tmpl (device) = frame 0's H header lines without trailing blanks or CR, each ended by '\n';
 * count_line (0 <= count_line < H) = the header line holding the atom count.  state (device int64[4], 8-byte aligned;
 * the caller sets {-u, INT64_MAX, 0, 0} before the first chunk, u = the lines of frame 0's UNITS pair, and keeps it
 * across chunks, which run in file order on one stream): [0] the running newline count minus u, [1] the atomic minimum
 * file offset of a CR not followed by LF, [2] one more than the largest frame number past frame_cap, [3] scratch.
 * Frame f >= 1 starts at line L = f P (lines counted from the first after the UNITS pair): frame_off[f] = its file
 * offset, status[f] = 0 when each ITEM line of its header equals tmpl's byte for byte (trailing blanks and CR allowed)
 * and its count line is natoms ([+-]digits between blanks), 1 when the host must decide -- a mismatch or a header that
 * runs past n_read (frame_off, status device, frame_cap entries).  frame_off[0] is set only with u > 0. */
int mkb_lammpstrj_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                        int64_t file_base, int64_t P, int64_t natoms, const uint8_t *tmpl, int64_t H,
                        int64_t count_line, int64_t *state, int64_t *frame_off, uint8_t *status, int64_t frame_cap);

/* K32: the header values of the LAMMPS dump frames that start in a chunk, parsed on the device after
 * mkb_lammpstrj_index on the same chunk, state and frame_off (same bytes, n, n_read, file_base and P).  Lines are
 * counted from the frame's first: step_line holds TIMESTEP ([+-] and at most 18 digits), time_line (-1: none) TIME,
 * box_line .. box_line + 2 the bound lines of 2 + ntilt values each (ntilt 0 or 1).  Frame f >= 1 of the chunk gets
 * step[f] (int64), time[f] (float64) and bounds[9 f + 3 i + j] (float64: line i's lo, hi and, with ntilt, tilt; 0
 * without), every value float() of its token (the grammar of mkb_xyz_decode); hstatus[f] = 1 when a line is left to
 * the host (another token or token count, or a line past n_read), its values then unspecified.  All device arrays of
 * frame_cap entries. */
int mkb_lammpstrj_head(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                       int64_t file_base, int64_t P, const int64_t *state, const int64_t *frame_off, int64_t frame_cap,
                       int64_t step_line, int64_t time_line, int64_t box_line, int64_t ntilt, int64_t *step,
                       double *time, double *bounds, uint8_t *hstatus);

/* K32: LAMMPS dump atom lines parsed on the device and placed by id; replaces the host reader's split(), float() and
 * int() per atom line, the sort by id and the transposition to the frame-minor arrays.  bytes = n_staged whole frames
 * of P = H + natoms lines back to back on the device (16-byte aligned, readable up to nbytes rounded up to 16), each
 * line ending in '\n' except possibly the last.  frame_of (HOST int32[n_frames]) = the staged frame of listed frame k.
 * role (device int8[n_cols]) = what column c of an atom line is: 0 skipped (its bytes < 0x80), 1 the id, 2-4 the
 * coordinate triple, 5-7 the image flags, 8-10 vx vy vz, 11-13 fx fy fz; columns past n_cols are not read.  ids NULL:
 * row = id - 1 (ids 1..natoms; without an id column row = the line's rank); else ids (device int64[natoms], ascending)
 * is searched for the row.  params (device float64[9 n_frames]): xlo ylo zlo lx ly lz xy xz yz of listed frame k.  Every
 * value is float() of its token in float64 (the grammar of mkb_xyz_decode; ids and image flags [+-] and at most 18
 * digits); with `scaled` x = ((xlo + xs lx) + ys xy) + zs xz, y = (ylo + ys ly) + zs yz, z = zlo + zs lz, with
 * `unwrap` x += (ix lx + iy xy) + iz xz, y += iy ly + iz yz, z += iz lz, each step a correctly rounded float64
 * operation, then one rounding to float32: coords (NULL: none) element (row, d, k) at coords[(row*3 + d)*frame_stride
 * + k]; vels and forces (NULL: none) the same layout.  fstat (device uint8, 4-byte aligned, n_frames rounded up to 4
 * entries; set to 0 here): bit 0 of fstat[k] when a line of listed frame k is left to the host (a short line, a token
 * outside the grammar, a byte >= 0x80, an undecided rounding), bit 1 when an id is unknown or seen twice; that frame's
 * rows are then unspecified. */
int mkb_lammpstrj_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                         const int32_t *frame_of, int64_t n_frames, int64_t natoms, int64_t H, const int8_t *role,
                         int64_t n_cols, const int64_t *ids, const double *params, int32_t scaled, int32_t unwrap,
                         float *coords, float *vels, float *forces, int64_t frame_stride, uint8_t *fstat);

/* K32: LAMMPS dump frames written on the device, the inverse of mkb_lammpstrj_decode for '%d %d %.9g %.9g %.9g'
 * lines.  coords float32 device, element (a, d, k) at coords[(a*3 + d)*frame_stride + k]; vels NULL or the same
 * layout.  ids, types (device int64[natoms]).  head (device) holds the n_frames frame headers back to back, frame k's at
 * [head_off[k], head_off[k + 1]) (head_off device int64[n_frames + 1], head_off[0] = 0, head_bytes = head_off[n_frames]).
 * Frame k is its header and then per atom '%d %d' of ids[a] and types[a], ' %.9g' of x, y, z (and with vels of vx, vy,
 * vz) and '\n', byte for byte Python's '%.9g' % float(v) (nan, inf, -inf as Python spells them), the frames back to
 * back from out.  A length pass, a scan and an emit pass: *total (device int64) receives the bytes written.  line_max
 * is the caller's bound on one atom line; head_bytes + n_frames*natoms*line_max > out_capacity is MKB_ERR_CAPACITY. */
int mkb_lammpstrj_encode(mkb_handle_t h, void *stream, const float *coords, const float *vels, int64_t frame_stride,
                         int64_t n_frames, int64_t natoms, const int64_t *ids, const int64_t *types, int64_t line_max,
                         const uint8_t *head, const int64_t *head_off, int64_t head_bytes, uint8_t *out,
                         int64_t out_capacity, int64_t *total);

/* K10 (SURVEY 8f row 3): the kernel of the `within` / `exwithin` atom selections, replaces within_distance
 * (moleculekit/atomselect_utils/atomselect_utils.pyx:612-653; called from atomselect/atomselect.py:243-251).
 * coords [n_atoms,3] float32 device (one frame, row-major); sel1 [n1] uint32 device = query atoms (NULL = all atoms,
 * n1 == n_atoms); sel2 [n2] uint32 device = source atoms; results [n1] uint8 device: results[ii] is SET to 1 when some
 * source atom lies at float32 squared distance < cutoff*cutoff of query ii and left untouched otherwise (the reference
 * only ever writes True).  Cell list over the source atoms instead of the reference's n1 x n2 loop; identical output. */
int mkb_within_distance(mkb_handle_t h, void *stream, const float *coords, int64_t n_atoms, const uint32_t *sel1,
                        int64_t n1, const uint32_t *sel2, int64_t n2, float cutoff, uint8_t *results);

/* K9 (SURVEY 8f row 4): orthorhombic wrapping of bonded groups, replaces wrap_box
 * (moleculekit/wrapping/wrapping.pyx:91-144; called from Molecule.wrap, moleculekit/molecule.py:2077).  t->coords is
 * MODIFIED IN PLACE like the reference's array.  groups [n_groups] uint32 device: ascending first-atom offsets of
 * consecutive groups, group g = atoms [groups[g], groups[g+1]) -- so n_groups - 1 ranges, the last entry (n_atoms in
 * Molecule.wrap) closes the last one.  centersel [n_centersel] uint32 device: atoms whose running-mean centre is the box
 * centre of each frame; when n_centersel == 0 the fixed `center` (HOST float[3]) is used instead (pyx:106-108).
 * float32 arithmetic with one rounding per operation and roundf half-away: bit-identical to the reference.  Index
 * ranges are the caller's responsibility (the reference compiles with boundscheck off as well). */
int mkb_wrap_box(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *groups, int64_t n_groups,
                 const uint32_t *centersel, int64_t n_centersel, const float *center);

/* K9b: wrapping of bonded groups in triclinic cells, replaces wrap_triclinic_unitcell (moleculekit/wrapping/wrapping.pyx:147-250,
 * unitcell = 2) and wrap_compact_unitcell (pyx:255-344 with get_pbc pyx:357-451 and pbc_dx pyx:454-505; unitcell = 0 is
 * its mode 0 "rectangular", 1 its mode 1 "compact") -- the calls Molecule.wrap makes when a box angle differs from 90
 * (moleculekit/molecule.py:2078-2090).  t->coords is MODIFIED IN PLACE (t->box is not used); boxvectors [3][3][stride]
 * float64 device, row i = box vector i, frame minor like Molecule.boxvectors.  groups / centersel / center as in
 * mkb_wrap_box; every atom is first centred on the wrap centre (also atoms outside all groups), then each group is
 * translated as the reference does it, float32 centres against float64 cell arithmetic: bit-identical coordinates.
 * Returns MKB_ERR_BAD_ARG "Too many triclinic vectors!!" where the reference raises that ValueError (pyx:439-441).  The
 * reference's unbounded while loops are capped at 2^20 iterations (only reached by cells without a positive diagonal). */
int mkb_wrap_triclinic(mkb_handle_t h, void *stream, const mkb_traj *t, const double *boxvectors,
                       int64_t bv_frame_stride, const uint32_t *groups, int64_t n_groups, const uint32_t *centersel,
                       int64_t n_centersel, const float *center, int32_t unitcell);

/* K12: hydrogen bonds over a trajectory, replaces hbonds.calculate (moleculekit/interactions/hbonds/hbonds.pyx:25-134; called
 * by hbonds_calculate, moleculekit/interactions/interactions.py:365-467).  donors [n_donors][2] uint32 device = (heavy atom,
 * hydrogen); acceptors [n_acceptors] uint32 device; sel1 / sel2 [n_atoms] uint32 device 0/1 flags; t->box is the
 * orthorhombic box (3, F).  intra != 0: both atoms in sel1 (pyx:70-73), else one in sel1 and the other in sel2
 * (pyx:74-77).  ignore_hs != 0: the heavy atom's distance is tested, no angle, hydrogen reported as -1 (pyx:101-105).
 * Two calls like K4 -- count: row_offsets [n_frames*n_donors + 1] int64 device = exclusive scan of the per-(frame, donor)
 * hit counts, *total_triples (HOST) the total (synchronises the stream); fill: triples [total][3] int32 device =
 * (heavy, hydrogen | -1, acceptor) in the reference's order (frame, donor, acceptor ascending).  Same booleans as the
 * reference binary (built as C++: round / sqrt / acos on float arguments are the float overloads), the acosf comparison as
 * a precomputed cosine bound. */
int mkb_hbonds_count(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *donors, int64_t n_donors,
                     const uint32_t *acceptors, int64_t n_acceptors, const uint32_t *sel1, const uint32_t *sel2,
                     float dist_threshold, float angle_threshold, int32_t intra, int32_t ignore_hs, int64_t *row_offsets,
                     int64_t *total_triples);
int mkb_hbonds_fill(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *donors, int64_t n_donors,
                    const uint32_t *acceptors, int64_t n_acceptors, const uint32_t *sel1, const uint32_t *sel2,
                    float dist_threshold, float angle_threshold, int32_t intra, int32_t ignore_hs,
                    const int64_t *row_offsets, int32_t *triples);

/* K13: ring-based interaction detectors over a trajectory.  mode 0 replaces pipi.calculate
 * (moleculekit/interactions/pipi/pipi.pyx:86-185), mode 1 cationpi.calculate (interactions/cationpi/cationpi.pyx:91-173),
 * mode 2 sigmahole.calculate (interactions/sigmahole/sigmahole.pyx:91-174); callers pipi_calculate / cationpi_calculate /
 * sigmahole_calculate (moleculekit/interactions/interactions.py:621-946).  rings_atoms uint32 device: concatenated ring atom
 * indexes; starts1 [n_rings1 + 1] uint32 device: ring start indexes of the first set.  second, uint32 device: mode 0 the start
 * indexes [n_second + 1] of the second ring set inside the same rings_atoms; mode 1 cation atom indexes [n_second]; mode 2
 * (halogen, bonded partner) pairs [n_second][2].  p0..p3: mode 0 dist_threshold1, angle_threshold1_max, dist_threshold2,
 * angle_threshold2_min; modes 1 / 2 dist_threshold, angle_threshold_min (p2, p3 unused).  Two calls like K4 -- count:
 * row_offsets [n_frames*n_rings1 + 1] int64 device, *total_pairs (HOST; synchronises the stream); fill: pairs [total][2]
 * int32 device = (ring index, second ring index | cation atom | halogen atom) and distangles [total][2] float32 device =
 * (distance, angle in degrees), in the reference's order (frame, ring, partner ascending).  Pairs and distances are the
 * reference binary's; the reported angle is within a few ulp (it comes from the device's acos, the reference's from glibc's
 * acosf).  Every ring must have at least 3 atoms: its normal comes from its first three.  The reference reads atoms of the
 * next ring (or past the end of rings_atoms) for a shorter ring, so it has no defined answer; the Python wrappers reject
 * one with a ValueError, and these entry points, which do not read the start indexes on the host, give it a zero normal
 * (dot products 0). */
int mkb_ring_pairs_count(mkb_handle_t h, void *stream, int32_t mode, const mkb_traj *t, const uint32_t *rings_atoms,
                         const uint32_t *starts1, int64_t n_rings1, const uint32_t *second, int64_t n_second, float p0,
                         float p1, float p2, float p3, int64_t *row_offsets, int64_t *total_pairs);
int mkb_ring_pairs_fill(mkb_handle_t h, void *stream, int32_t mode, const mkb_traj *t, const uint32_t *rings_atoms,
                        const uint32_t *starts1, int64_t n_rings1, const uint32_t *second, int64_t n_second, float p0,
                        float p1, float p2, float p3, const int64_t *row_offsets, int32_t *pairs, float *distangles);

/* K14: trajectory superposition, replaces the frame loop of Molecule.align (moleculekit/align.py, _pp_align and
 * _pp_measure_fit) and the RMSD of MetricRmsd (moleculekit/projections/metricrmsd.py, molRMSD).  All pointers except
 * the mkb_traj structs are device pointers.  t is the trajectory; ref (its box is not used) has either 1 frame (every frame
 * is fitted to it) or t->n_frames frames (frame f is fitted to reference frame f: matchingframes).  sel / refsel [n_sel]
 * uint32 = the atoms of t and of ref that correspond, pairwise; n_sel == 0 is MKB_ERR_BAD_ARG.  frames [n_frames] uint32
 * = the listed frames of t, distinct (NULL = every frame, n_frames ignored); item k of the list is frame frames[k], and
 * the per-frame outputs below are indexed by k.  Frames not in the list are never touched.  Index ranges of sel, refsel
 * and frames are the caller's responsibility.
 *
 * fit:   records [n][16] float64 = R (3x3 row-major), p_bar (3), q_bar (3), one pad; the optimal proper rotation of the
 *        centred selection of frame frames[k] onto the centred reference (Kabsch, det R = +1, H = 0 gives the
 *        identity), so that x' = R (x - p_bar) + q_bar.  Centroids and covariance are summed in float64 in an order that
 *        depends only on the selection (a frame gives the same bits whatever else is in the call); the rotation comes
 *        from Horn's quaternion matrix by cyclic Jacobi in float64.  status [n] int32: 0 = ok, 1 = non-finite
 *        covariance or centroid (NaN / inf in a selected coordinate; the record then holds R = identity).
 * apply: t->coords is MODIFIED IN PLACE: every atom of every listed frame with status 0 (status NULL = all) becomes
 *        fl32(R (x - p_bar) + q_bar) evaluated in float64 -- within 1 float32 ulp of the float64 superposition.
 * rmsd:  out [n] float32 = sqrt(mean over the selection of |T_k(x) - q|^2) in float64, T_k = the fit record k
 *        (records NULL = no transform: plain molRMSD).
 * The handle's timing events (mkb_set_timing) bracket the reference centring (prep) and the fit / apply / RMSD kernels
 * (main). */
int mkb_align_fit(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref,
                  const uint32_t *refsel, int64_t n_sel, const uint32_t *frames, int64_t n_frames, double *records,
                  int32_t *status);
int mkb_align_apply(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *frames, int64_t n_frames,
                    const double *records, const int32_t *status);
int mkb_rmsd(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref,
             const uint32_t *refsel, int64_t n_sel, const uint32_t *frames, int64_t n_frames, const double *records,
             float *out);

/* K15: aligned coordinate features and per-atom fluctuations, replace the host gather of MetricCoordinate
 * (moleculekit/projections/metriccoordinate.py) and the squared deviations of MetricFluctuation
 * (moleculekit/projections/metricfluctuation.py).  All pointers except the mkb_traj struct are device pointers.  sel
 * [n_sel] uint32 = the selected atoms of t in output order; n_sel == 0 is MKB_ERR_BAD_ARG.  frames [n_frames] uint32 = the
 * listed frames of t (NULL = every frame, n_frames ignored); item k of the list is frame frames[k] and output row k
 * belongs to it.  records [n][16] float64 = the K14 fit records of mkb_align_fit, record k for item k (NULL = no
 * transform).  The aligned coordinate c is fl32(R (x - p_bar) + q_bar) evaluated in float64: the bits mkb_align_apply
 * writes in place.  The trajectory is not modified.  Index ranges of sel, frames and group_offsets are the caller's
 * responsibility.
 *
 * coordinates:  out[k * ld_out + d * n_sel + i] float32 = c_d of atom sel[i] in item k (one row per listed frame, all X
 *               of the selection, then all Y, then all Z); ld_out >= 3 n_sel, so a frame shard can write into the rows
 *               of a larger matrix, and the row block into the columns of a wider one.
 * coord_sums:   sums[i * 3 + d] float64 = sum over the listed frames of c_d of atom sel[i] (zero without frames), added in
 *               list order within fixed chunks of 64 items and the chunks in order: the bits depend only on the
 *               selection and the ordered frame list (a frame slice gives the bits of the same explicit list).
 * fluctuation:  centre [n_sel][3] float64 = the point each selected atom deviates from (the mean, or a reference).
 *               Without group_offsets: out[k * ld_out + i] float32 = fl32(sum_d (c_d - centre[i][d])^2), the sum in
 *               float64 (no fused multiply-add, axis order); ld_out >= n_sel.  With group_offsets [n_groups + 1] int64
 *               (0 = first, n_sel = last, nondecreasing; a group is the selection positions [off[g], off[g+1]), empty
 *               groups give NaN): out[k * ld_out + g] = fl32(the float64 mean of the group's unrounded per-atom values,
 *               added in selection order); ld_out >= n_groups.  c is recomputed from the trajectory, never read back.
 * The handle's timing events (mkb_set_timing) bracket the kernels (main; prep is empty). */
int mkb_coordinates(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                    const uint32_t *frames, int64_t n_frames, const double *records, float *out, int64_t ld_out);
int mkb_coord_sums(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                   const uint32_t *frames, int64_t n_frames, const double *records, double *sums);
int mkb_fluctuation(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                    const uint32_t *frames, int64_t n_frames, const double *records, const double *centre,
                    const int64_t *group_offsets, int64_t n_groups, float *out, int64_t ld_out);

/* K20: weighted per-frame moments of atom groups, replace the per-frame centres and spreads of MetricGyration
 * (moleculekit/projections/metricgyration.py) and MetricSphericalCoordinate
 * (moleculekit/projections/metricsphericalcoordinate.py) after the reference's align.  t, sel, frames and records as for
 * the K15 entry points above (device pointers; c = the aligned float32 coordinate).  weights [n_sel] float64 and
 * group_offsets [n_groups + 1] int64 are HOST arrays (they size the launch): group g is the selection positions
 * [off[g], off[g+1]); the offsets run from 0 to n_sel and increase strictly (no empty group); weights NULL = all 1; a
 * group whose weights do not sum to a finite value > 0 is MKB_ERR_BAD_ARG.  Every check is made before any work is
 * enqueued; the call returns once both arrays have been copied.
 *
 * out [n][n_groups][6] float64 (device), W the group's weight total:
 *   out[(k n_groups + g) 6 + d]     = mu_d = sum w c_d / W
 *   out[(k n_groups + g) 6 + 3 + d] = v_d = sum w (c_d - mu_d)^2 / W, per axis (never negative)
 * The sums run in float64 relative to the group's first position in the same frame, within segments of at most 512
 * positions that depend only on the group sizes, added in a fixed order: the bits of a frame's row depend only on the
 * selection, groups and weights (not on the grid, the frame slice or the rest of the frame list).  A non-finite
 * coordinate in a group gives NaN in all six values of that (item, group) only.  The handle's timing events bracket the
 * kernels (main; prep is empty). */
int mkb_frame_moments(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                      const uint32_t *frames, int64_t n_frames, const double *records, const double *weights,
                      const int64_t *group_offsets, int64_t n_groups, double *out);

/* K16: torsion angles, replace the per-dihedral loop of MetricDihedral (moleculekit/projections/metricdihedral.py over
 * moleculekit.dihedral.dihedralAngle).  All pointers except the mkb_traj struct are device pointers.  quads [n_quads][4]
 * int32 = atom rows of t (p0, p1, p2, p3 of each dihedral), 16-byte aligned; n_quads == 0 is MKB_ERR_BAD_ARG.  frames
 * [n_frames] uint32 = the listed frames of t (NULL = every frame, n_frames ignored); item k of the list is frame
 * frames[k] and output row k belongs to it.  Index ranges of quads and frames are the caller's responsibility.  The
 * coordinates are used as given (no minimum image), and nothing about the trajectory's orientation is needed.
 *
 * Per (item, quadruple), in float64 from the float32 points: b0 = p0 - p1, b1 = p2 - p1, b2 = p3 - p2, u = b1 / |b1|,
 * v = b0 - (b0.u) u, w = b2 - (b2.u) u, x = v.w, y = (u x v).w.  The sign is IUPAC's: looking along p1 -> p2 the angle
 * is positive when p1-p0 turns clockwise onto p2-p3 (cis 0, trans +-pi).
 *   sincos == 0:  out[k * ld_out + j] float32 = fl32(atan2(y, x)), radians; ld_out >= n_quads.
 *   sincos == 1:  out[k * ld_out + 2 j] = fl32(y / hypot(x, y)) (sine), out[k * ld_out + 2 j + 1] = fl32(x / hypot(x, y))
 *                 (cosine); ld_out >= 2 n_quads.
 * A degenerate quadruple -- b0 x b1 or b1 x b2 exactly zero, each component a[i] b[j] - a[j] b[i] evaluated in float64
 * without a fused multiply-add (p0, p1, p2 or p1, p2, p3 collinear in any orientation, or p1 == p2) -- gives angle 0 and
 * (sin, cos) = (0, 1); a non-finite coordinate among the four points gives NaN.  ld_out lets a frame shard write into the rows of a
 * larger matrix.  The handle's timing events (mkb_set_timing) bracket the kernel (main; prep is empty). */
int mkb_dihedrals(mkb_handle_t h, void *stream, const mkb_traj *t, const int32_t *quads, int64_t n_quads,
                  const uint32_t *frames, int64_t n_frames, int32_t sincos, float *out, int64_t ld_out);

/* K17: Shrake-Rupley solvent-accessible surface area, replaces mdtraj's per-frame asa_frame loop that moleculekit's
 * MetricSasa calls.  All pointers except the mkb_traj struct are device pointers.  env [n_env] uint32 = atom rows of t
 * that form the environment (the reference's filtersel); radii [n_env] float32 = radius plus probe in nm, finite and
 * > 0; query [n_query] uint32 = positions in env of the atoms whose area is computed; sphere [n_sphere][3] float32 =
 * unit sphere points, 1 <= n_sphere <= 65536.  frames [n_frames] uint32 = the listed frames of t (NULL = every frame,
 * n_frames ignored); output row k belongs to item k.  Index ranges are the caller's responsibility.  No wrapping and no
 * minimum image.
 *
 * Per item, every operation float32 and rounded on its own (no fused multiply-add): x_nm = fl(x / 10); env atom j is
 * a neighbour of query atom i when j != i and fl(fl(fl(dx dx) + fl(dy dy)) + fl(dz dz)) < fl(fl(R_i + R_j)^2), dx =
 * fl(x_i - x_j); sphere point s of i sits at p = fl(x_i + fl(R_i s)) and is buried when the same sum over fl(p - x_k)
 * is < fl(R_k R_k) for some neighbour k; n_i = the points not buried; a_i = fl(fl(fl(c R_i) R_i) n_i) nm^2 with
 * c = (float)(4 pi / n_sphere).  A non-finite coordinate takes part in no neighbour relation.
 *   group_offsets NULL:  out[k * ld_out + q] = fl(a_q 100) (Angstrom^2); ld_out >= n_query.
 *   group_offsets [n_groups + 1] int64 (query positions, non-decreasing, first 0, last n_query):
 *                        out[k * ld_out + g] = fl(s 100), s = the a_q of group g added in order to a float32 zero;
 *                        ld_out >= n_groups.
 * status [1] int64, 8-byte aligned: -1 when no query atom has an env atom j != i with d2 < 1e-10 nm^2 (coincident
 * atoms, where the reference exits), else (item << 32) | q of the first such item and query (smallest key).  The
 * listed frames are processed in chunks of mkb_sasa_chunk_frames(n_env, n_query, n_groups) items (0 with groups
 * absent means n_groups = 0), so scratch stays bounded.  The handle's timing events bracket the whole call (main; prep
 * is empty). */
int mkb_sasa(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *env, int64_t n_env, const float *radii,
             const uint32_t *query, int64_t n_query, const int64_t *group_offsets, int64_t n_groups,
             const float *sphere, int32_t n_sphere, const uint32_t *frames, int64_t n_frames, float *out,
             int64_t ld_out, int64_t *status);
int64_t mkb_sasa_chunk_frames(int64_t n_env, int64_t n_query, int64_t n_groups);

/* K18: DSSP secondary structure, replaces mdtraj's compute_dssp (a port of DSSP 2.2.0) that moleculekit's
 * MetricSecondaryStructure calls per frame.  All pointers except the mkb_traj struct are device pointers.  backbone
 * [n_res][4] int32 = atom rows of t of the N, CA, C and O of every residue of the DSSP sequence (all chains
 * concatenated, indexed 0..n_res-1), 1 <= n_res <= 2^28; flags [n_res] uint8: bit 0 = proline, bit 1 = the residue
 * differs in chain or segid from the previous one.  frames [n_frames] uint32 = the listed frames of t (NULL = every
 * frame, n_frames ignored); item k is frame frames[k].  Index ranges are the caller's responsibility.  No minimum image.
 *
 * Per item, everything in float64 from the float32 Angstrom coordinates, every operation rounded on its own (no fused
 * multiply-add); dist(a, b) = sqrt((dx dx + dy dy) + dz dz), d = a - b.
 *   breaks   between r and r + 1 when bit 1 of flags[r + 1] is set or dist(C_r, N_r+1) > 2.5 (a NaN distance is not a
 *            break); NoChainBreak(a, b) = no break between consecutive residues of [a, b].
 *   H        H_r = N_r + v / |v| per component, v = C_r-1 - O_r-1, when r is not proline, r > 0 and no break lies
 *            between r - 1 and r; else H_r = N_r.
 *   energy   E(d, a) for donor d (N-H) and acceptor a (C=O), evaluated when a != d, a != d - 1, d is not proline and
 *            dist(CA_d, CA_a) < 9.0: -9.9 when one of dHO, dHC, dNC, dNO is < 0.5, else
 *            ((K/dHO - K/dHC) + K/dNC) - K/dNO with K = -27.888; then E = round(E 1000) / 1000 (half away from zero)
 *            and E = -9.9 where E < -9.9.  Each donor keeps two slots (partner, energy), initially (-1, 0.0), filled in
 *            ascending acceptor order: E < slot0.E shifts slot 0 to slot 1 and takes slot 0, else E < slot1.E takes
 *            slot 1 (the stable top two by (E, index) among E < 0).  TestBond(x, y) = a slot of x holds y with E < -0.5.
 *   bend     residue i with i - 2, i + 2 in range and NoChainBreak(i - 2, i + 2): u = CA_i - CA_i-2,
 *            w = CA_i+2 - CA_i, x = (u.u)(w.w), c = (u.w) / sqrt(x) if x > 0 else 0; bent when c < bend_cos, the
 *            smallest double c with acos(c) 180 / pi <= 70 (found on the host against libm).
 *   codes    DSSP 2.2.0's helix flags (strides 3, 4, 5), bridges (i, j >= i + 3) with its grouping and ladder merge in
 *            its order, uint32 differences included, then E / B, H, G, I (no pi-helix priority), T and S.
 *            codes[k * ld + r] uint8: 0 loop, 1 H, 2 B, 3 E, 4 G, 5 I, 6 T, 7 S; ld >= n_res.
 * hb_partner [item][n_res][2] int32 and hb_energy [item][n_res][2] float64 (both NULL, or both given) receive both
 * slots of every donor.  Per-frame state lives in global scratch (no residue limit in shared memory); the listed frames
 * are processed in chunks of mkb_dssp_chunk_frames(n_res) items, so scratch stays bounded.  The handle's timing events
 * bracket the whole call (main; prep is empty). */
int mkb_dssp(mkb_handle_t h, void *stream, const mkb_traj *t, const int32_t *backbone, const uint8_t *flags,
             int64_t n_res, double bend_cos, const uint32_t *frames, int64_t n_frames, uint8_t *codes, int64_t ld,
             int32_t *hb_partner, double *hb_energy);
int64_t mkb_dssp_chunk_frames(int64_t n_res);

/* K19: TM-score, replaces the superposition search of the TMscore program (Zhang & Skolnick, Proteins 2004) that
 * moleculekit's molTMscore runs per frame.  All pointers except the mkb_traj structs, frag and the scalars are device
 * pointers.  Pair k (0 <= k < L = n_pairs, 1 <= L <= mkb_tmscore_max_pairs()) joins atom row sel[k] of t (model x_k) and
 * atom row refsel[k] of frame 0 of ref (reference y_k).  l_norm >= 1 is the normaliser.  d0 > 0, d0_search and frag
 * [n_frag] host int32 (1 <= n_frag <= 6, each in [1, L]) are computed by the caller: d0 = 0.5 if l_norm <= 15, else
 * max(0.5, 1.24 pow(l_norm - 15, 1/3) - 1.8); d0_search = d0 clamped to [4.5, 8]; frag = floor(L / 2^i) for i = 0..4
 * while it is > min(4, L), then min(4, L).  frames [n_frames] uint32 = the listed frames of t (NULL = every frame,
 * n_frames ignored); item k is frame frames[k].  Index ranges are the caller's responsibility.
 *
 * Per item, everything in float64 from the float32 coordinates, every operation rounded on its own (no fused
 * multiply-add), every sum sequential in ascending pair order:
 *   fit      of a pair set of size c: p = (sum x) / c, q = (sum y) / c, H[a][b] = sum (x_a - p_a)(y_b - q_b) in a second
 *            pass; R = the rotation of Horn's quaternion (the eigenvector of the largest eigenvalue of the symmetric 4x4
 *            matrix by cyclic Jacobi, at most 50 sweeps, the "late" threshold after sweep 3, ties to the lowest index);
 *            x' = R (x - p) + q, each row ((R0 a0 + R1 a1) + R2 a2) + q.
 *   score    over all L pairs: dis = sqrt((dx dx + dy dy) + dz dz), d = x' - y, t = dis / d0; S = (sum 1 / (1 + t t)) /
 *            l_norm.
 *   cut      the pairs with dis < dcut; while fewer than 3 and L > 3, dcut (a local copy) grows by 0.5 and the pairs are
 *            cut again, at most 2^20 times.
 *   search   for every fragment length Li in order and every start iL = 0..L - Li: fit the pairs iL..iL + Li - 1 and
 *            cut at d0_search - 1; then up to 20 times: stop if the cut set is empty, fit the cut set, cut at
 *            d0_search + 1, stop if the new set equals the one just fitted.
 *   output   tm[k] = the largest S of every fit of every seed; rmsd[k] = sqrt((sum |x' - y|^2) / L) under the first
 *            fit (the all-pairs one).  A non-finite coordinate among the pairs gives NaN for both, in that item only.
 * Two bitmasks of L bits per resident thread live in global scratch.  The handle's timing events bracket the kernel
 * (main; prep is empty). */
int mkb_tmscore(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref,
                const uint32_t *refsel, int64_t n_pairs, int64_t l_norm, double d0, double d0_search,
                const int32_t *frag, int32_t n_frag, const uint32_t *frames, int64_t n_frames, double *tm,
                double *rmsd);
int64_t mkb_tmscore_max_pairs(void);

/* K27: TM-align, replaces the TM-align program (Zhang & Skolnick, Nucleic Acids Res. 2005) that moleculekit's
 * molTMalign runs per frame: a sequence-independent residue alignment and superposition of x, the mol CA trace (atom
 * rows sel[0..xlen) of t), onto y, the reference trace (atom rows refsel[0..ylen) of ref).  All pointers except the
 * mkb_traj structs and params are device pointers.  5 <= xlen, ylen <= mkb_tmalign_max_residues() (TM-align's "too
 * short" below 5).  ref_per_frame = 0: every item against frame 0 of ref; 1: item k against frame f of ref, f its own
 * listed frame (ref n_frames >= t n_frames).  frames [n_frames] uint32 = the listed frames of t (NULL = every frame).
 * Index ranges are the caller's responsibility.  The restatement is tests/tmalign_oracle.c, in the shape of the C++
 * release's TMalign_main; invmap[j] is the x residue aligned to y residue j, or -1; dist is the SQUARED distance.
 *
 * params [10] host float64 (tmalign_parameters, C pow): Lnorm = min(xlen, ylen); d0 = 0.168 if Lnorm <= 19 else
 * 1.24 (Lnorm - 15)^(1/3) - 1.8; D0_MIN = d0 + 0.8 and d0 = D0_MIN; d0_search = d0 clamped to [4.5, 8]; score_d8 =
 * 1.5 Lnorm^0.3 + 3.5; ddcc = 0.1 if Lnorm <= 40 else 0.4; dcu0 = 4.25: [d0, d0_search, score_d8, D0_MIN, ddcc,
 * dcu0], then the final d0 (0.5 if L <= 21 else the same formula, floored at 0.5) and its clamped d0_search for
 * L = ylen, then for L = xlen.
 *
 * Per item, everything in float64 from the float32 coordinates, every operation rounded on its own (no fused
 * multiply-add), every sum sequential in pair order:
 *   fit       K19's: two-pass centroids p, q and H, Horn's quaternion by cyclic Jacobi; x' = R (x - p) + q, each row
 *             ((R0 a0 + R1 a1) + R2 a2) + q with a = x - p; dist = (dx dx + dy dy) + dz dz.  An empty set fits the
 *             identity.
 *   sec       residue i with i - 2, i + 2 in range: the square roots d13 d14 d15 d24 d25 d35 over i - 2 .. i + 2; H when
 *             |d15 - 6.37|, |d14 - 5.18|, |d25 - 5.18|, |d13 - 5.45|, |d24 - 5.45|, |d35 - 5.45| are all < 2.1, else E
 *             against 13, 10.4, 10.4, 6.1, 6.1, 6.1 and 1.42, else T when d15 < 8, else C (also without neighbours).
 *   score_fun8  cut at dist < (d + inc 0.5)^2, inc = 0, 1, ... while fewer than 3 pairs and n > 3; method 8 sums
 *             1 / (1 + dist / d0^2) over pairs with dist <= score_d8^2, method 0 over all; divided by Lnorm (the
 *             standard form: by n).
 *   TMscore8_search  over n pairs: fragment lengths n >> i while > min(4, n), then min(4, n) (at most 6); starts 0,
 *             +simplify_step, the last start n - L always; each start: seed fit, cut at d0_search - 1, then up to 20
 *             refits of the cut set cut at d0_search + 1, stopping on an empty set or a repeated one; the best score
 *             (strict >) and its fit.  An empty pair set scores 0 with the identity.
 *   get_score_fast  fit all pairs of the map, score; refit dist <= d0_search^2 (+0.5 while < 3 pairs and n > 3) and,
 *             when that set is not all pairs, once more at d0_search^2 + 1; the largest of the three (>=).
 *   NWDP_TM   value d = val[i-1][j-1] + term (1 / (1 + dist / d02) under a fit; that + 0.5 where the codes match;
 *             1 where they match), h / v = the neighbour + gap_open when that neighbour took its diagonal; the
 *             diagonal when d >= h && d >= v, else v when v >= h, else h; traceback from (xlen, ylen) by the same rule.
 *   DP_iter   for gap_open in {-0.6, 0}[g1..g2), up to the iteration count: DP under the current fit with d02 = d0^2,
 *             detailed_search (simplify_step 40, method 8) whose fit is the next one; keep the best map (>); stop when
 *             |TM_old - TM| < 1e-6 (TM_old is carried across the gap opens).
 *   initial   1 gapless threading over every shift, min_ali = max(5, min_len / 2), best shift on >=; DP_iter(0, 2, 30).
 *             2 DP on the codes, gap -1; DP_iter(0, 2, 30) if TM > 0.2 TMmax.  3 get_initial5: fragment lengths {20,
 *             100} capped at aL / 3, aL / 2, jumps 45 / 35 / 25 / 15 for lengths > 250 / > 200 / > 150 / else, capped
 *             at len / 3; per fragment pair a fit, DP with gap 0 and d01 = max(d0 + 1.5, D0_MIN), get_score_fast, first
 *             maximum (>) wins; DP_iter(0, 2, 2) if TM > ddcc TMmax.  4 the score 1 / (1 + dist / d01^2) (+ 0.5 where
 *             the codes match) under the fit of the best map, gap -1; DP_iter(0, 2, 30) if TM > ddcc TMmax.  5
 *             find_max_frag on both traces (cutoff dcu0 grown by a running product of 1.1 until the longest run of
 *             consecutive dist < cutoff^2 has min(4, len / 3) residues), the x fragment when Lx < Ly or Lx == Ly and
 *             xlen <= ylen, else the y one, trimmed to [floor(0.1 L0), floor(0.89 L0)] when it spans L0 =
 *             min(xlen, ylen), threaded with min_ali = max(3, floor(min_len / 2.5)), best on >=; DP_iter(1, 2, 2) if
 *             TM > ddcc TMmax.  Each initial map first goes through detailed_search (40, method 8); TMmax and the
 *             best map update on strict >.
 *   final     detailed_search_standard (simplify_step 1, method 8) on the best map; under its fit the aligned pairs
 *             with sqrt(dist) <= score_d8 are the nali final pairs (invmap keeps only them); rmsd = sqrt(sum dist /
 *             nali) under the fit of those pairs; tm[k][0] = TMscore8_search (simplify_step 1, method 0) over them
 *             with the final parameters of L = ylen, whose best fit is records[k]; tm[k][1] the same for L = xlen.
 *             nali = 0 gives scores and rmsd 0 and the identity record.
 * Outputs per item k: tm [n][2], rmsd [n], nali [n] int32, invmap [n][ylen] int32, records [n][16] in K14's layout
 * (R row-major, p, q, pad; mkb_align_apply moves frames with them).  A non-finite selected coordinate (of the frame or
 * its reference frame) gives NaN scores and rmsd, nali 0, invmap all -1 and the identity record, in that item only.
 * Not confirmed against TMalign.cpp (no source at hand): the fit (the program uses its own Kabsch routine), the
 * running product in place of pow(1.1, inc), the 2019 release's extra tie search for Lx == Ly and xlen == ylen (left
 * out), the final search's simplify_step, and that the alignment reported is the score_d8-filtered map.
 * One warp per item; per-item state in global scratch, items in chunks of mkb_tmalign_chunk_frames(xlen, ylen).
 * The handle's timing events bracket the launches (main; prep is empty). */
int mkb_tmalign(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t xlen, const mkb_traj *ref,
                const uint32_t *refsel, int64_t ylen, int32_t ref_per_frame, const double *params,
                const uint32_t *frames, int64_t n_frames, double *tm, double *rmsd, int32_t *nali, int32_t *invmap,
                double *records);
int64_t mkb_tmalign_max_residues(void);
int64_t mkb_tmalign_chunk_frames(int64_t xlen, int64_t ylen);

#ifdef __cplusplus
}
#endif
#endif /* MKB200_H */
