/*
 * lidiff_b200 — C ABI of the H100-native (sm_90a) implementation of the LiDiff denoising hot path.
 *
 * The reference (PRBonn/LiDiff) reaches this path through three un-vendored Python packages, not
 * through a C interface (SURVEY.md 8b):
 *     import MinkowskiEngine as ME      lidiff/models/minkunet.py:6, tools/diff_completion_pipeline.py:2
 *     pykeops.torch.LazyTensor.argKmin  lidiff/models/minkunet.py:8,412-416
 *     diffusers.DPMSolverMultistepScheduler.step   tools/diff_completion_pipeline.py:6,163
 * Each entry point below names the reference call site(s) it stands behind.  The Python operator
 * surface that mirrors those packages lives in lidiff_b200/ and binds this library with ctypes
 * (INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - every buffer is CALLER-OWNED device memory (a torch CUDA tensor); the library allocates nothing
 *     the caller can see and keeps no state besides the handle's error string;
 *   - all calls are asynchronous on the given `stream` (a cudaStream_t passed as void*), never
 *     synchronise, never allocate => capturable in a CUDA graph;
 *   - data-dependent row counts live in DEVICE int32 scalars (`d_n*`); buffers are sized by a host
 *     capacity (`*_cap`) and kernels read the count on the device;
 *   - return value: 0 = OK, negative = error; `lb2_last_error(h)` gives the message;
 *   - coordinates are int32 rows [b, x, y, z]; features are fp32 row-major (rows, channels);
 *   - no CPU fallback exists: without a CUDA device the calls fail with LB2_ERR_CUDA.
 */
#ifndef LIDIFF_B200_H_
#define LIDIFF_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LB2_OK            0
#define LB2_ERR_ARG      -1
#define LB2_ERR_CUDA     -2
#define LB2_ERR_UNSUP    -3

#define LB2_KEY_EMPTY 0xFFFFFFFFFFFFFFFFull

/* ---- handle ----------------------------------------------------------------------------------- */
int         lb2_create(int device, void** handle);
void        lb2_destroy(void* handle);
const char* lb2_last_error(void* handle);
int         lb2_version(void);
/* number of kernels this library has launched through `handle` since creation (bench gpu_launches) */
int64_t     lb2_launch_count(void* handle);
/* synchronising read-and-clear of the device status word; bit0 = a coordinate fell outside the key
 * range (batch in [0, 1023], every axis in [-131072, 131071]) or was NaN, and its key was clamped into
 * the range.  Returns the word (>= 0) or an error. */
int         lb2_read_status(void* handle, void* stream);

/* ---- hash grid (coordinate manager)  — replaces ME's CoordinateManager -------------------------
 * One hash grid per coordinate level.  `keys` (uint64[cap_table]) and `vals` (int32[2*cap_table]:
 * [0,cap) scratch "first point index", [cap,2cap) row id) are caller-owned; cap_table is a power
 * of two >= 2 * max rows.  Key packing: 10 bit batch | 3 x 18 bit signed coordinate, so the key range is
 * batch in [0, 1023] and every axis in [-131072, 131071].  The range is closed under the stride maps' floor
 * to multiples of 2^l: a level-0 row in range has every coarser row in range.  A kernel-map neighbour outside
 * the range is a miss (nothing wraps).
 */
typedef struct {
    uint64_t* keys;
    int32_t*  vals;
    int32_t   cap_table;
} lb2_grid;

/* coord = round_half_even(x / resolution) on every column of an (n,ncol) fp32 array.
 * Reference: tools/diff_completion_pipeline.py:71-72, utils/collations.py:8-12 (torch.round(x/res)).
 * div_mode 0: true fp32 division; 1: multiply by fp32(1/resolution) (PyTorch CUDA scalar division). */
int lb2_quantize(void* h, void* stream, const float* x, int64_t n_elem, float resolution, int div_mode,
                 float* out_coord);

/* ME.TensorField.sparse() coordinate part (pipeline:149, minkunet.py:135,597) and ME strided
 * coordinate maps (conv stride 2, minkunet.py:103,184...).
 * Input rows: either fp32 integer-valued coords (`in_f`, floor() is applied; TensorField) or int32
 * coords (`in_i`; a parent level).  If ts_floor > 0 the xyz columns are floored to multiples of
 * ts_floor (stride map).  Output: unique rows in FIRST-OCCURRENCE order, `inverse[i]` = output row of
 * input row i, `*d_nout` = number of unique rows.  `scratch` >= lb2_unique_scratch_bytes(n_cap).
 * n_cap <= 4194304 (4M rows; larger: LB2_ERR_ARG).  Rows past min(*d_nin, n_cap) are not read.
 * Non-finite in_f values: +-inf and values beyond the int32 range convert to INT_MIN / INT_MAX, NaN to 0; such a
 * row (a NaN in any column, or any column outside the key range) raises status bit 0 (lb2_read_status) and is
 * grouped under its clamped key, so the caller must treat the build as failed. */
size_t lb2_unique_scratch_bytes(int64_t n_cap);
int lb2_unique_build(void* h, void* stream,
                     const float* in_f, const int32_t* in_i, const int32_t* d_nin, int32_t n_cap,
                     int32_t ts_floor, lb2_grid grid,
                     int32_t* out_coords, int32_t* inverse, int32_t* d_nout, void* scratch);

/* UNWEIGHTED_AVERAGE voxel features (ME.SparseTensorQuantizationMode, pipeline:77): mean of member
 * point features, out (m_cap, c).  Every member is rounded to a fixed-point quantum 2^-s and summed exactly in int64, so the
 * result does not depend on the order of the points.  For a (row, channel) with n members, largest magnitude in
 * [2^(e-1), 2^e), s = 61 - e - bitlen(n) and exact mean m:
 *     |out - m| <= ulp32(m)/2 + 2^-(s+1) + 2^-50 |m|,
 * and out = RN32(m) wherever m is farther than 2^-(s+1) + 2^-50 |m| from an fp32 rounding midpoint (2^-(s+1) is about
 * 2^-51 of the largest member for a 1000-member voxel).  Rows whose members are all zero are +0; a row with a NaN or +-inf
 * member is NaN in that channel (ME's fp32 sum would give +-inf for an inf member), as is a row with no members;
 * rows [*d_m, m_cap) are 0.  `scratch` >= lb2_voxel_mean_scratch_bytes(m_cap, c) bytes. */
size_t lb2_voxel_mean_scratch_bytes(int32_t m_cap, int32_t c);
int lb2_voxel_mean(void* h, void* stream, const float* feats, const int32_t* inverse, int32_t n,
                   int32_t c, const int32_t* d_m, int32_t m_cap, float* out, void* scratch);

/* Kernel map (ME kernel maps for MinkowskiConvolution / ConvolutionTranspose; minkunet.py:17-24,36-42).
 * Output-stationary neighbour table: nbr[k * nbr_stride + o] = input row at coords(o) + offset_k, or -1.
 *   ks=3: offset_d = (k_d - 1) * step      ks=2: offset_d = k_d * step   (step < 0: transposed map)
 *   k = kx + ks*ky + ks*ks*kz.
 * pair_count (device uint64, optional): += number of (in,out) pairs found (roofline accounting).
 * row_mask (uint32[nout_cap], optional): bit k of row_mask[o] set iff nbr[k][o] >= 0. */
int lb2_kernel_map(void* h, void* stream, lb2_grid grid_in, const int32_t* out_coords,
                   const int32_t* d_nout, int32_t nout_cap, int32_t ks, int32_t step,
                   int32_t* nbr, int64_t nbr_stride, uint64_t* pair_count, uint32_t* row_mask);

/* The 3^3 stride-1 map of a coordinate set onto itself (`grid` was built from exactly `coords`; step = the level's tensor stride):
 * same table and row masks as lb2_kernel_map(ks = 3), with half the hash probes (the pair set is symmetric: row j at offset k of row o
 * <=> o at offset 26 - k of j). */
int lb2_kernel_map_self(void* h, void* stream, lb2_grid grid, const int32_t* coords, const int32_t* d_n, int32_t n_cap,
                        int32_t step, int32_t* nbr, int64_t nbr_stride, uint64_t* pair_count, uint32_t* row_mask);

/* Execution order of the output rows for lb2_spconv_forward (no reference counterpart: scheduling only).
 * perm[0..n) = the rows 0..n-1 sorted by their neighbour mask (kvol 27: centre-only rows, rows with one neighbour grouped
 * by it, then the rest in mask order; kvol <= 8: by the 8-bit mask) so that 128-row tiles skip unpopulated kernel offsets.
 * Results do not depend on the order.  scratch >= lb2_row_order_scratch_bytes(n_cap).
 * coords (optional, kvol 27 only): the rows' int32 [b,x,y,z] coordinates; rows of equal mask are then ordered by the Morton code of
 * (x,y,z) >> coord_shift (coord_shift = log2 of the level's tensor stride), which makes the tiles of large mask groups spatially
 * compact (L2 locality of the gathers).  The sort is stable: rows of equal key (and Morton code) keep their index order, so
 * the order, and with it the tensor-core convolution's per-tile accumulation grouping, is the same on every run. */
size_t lb2_row_order_scratch_bytes(int32_t n_cap);
int lb2_row_order(void* h, void* stream, const uint32_t* row_mask, const int32_t* d_n, int32_t n_cap,
                  int32_t kvol, int32_t* perm, void* scratch, const int32_t* coords, int32_t coord_shift);

/* Cost order of the tiles of a map (scheduling only; results do not depend on it): order128[i] / order256[i] = index of the i-th most
 * expensive 128-row tile / 256-row super-tile of the row order `row_perm`, cost = number of kernel offsets the tile has to run (popcount of
 * the OR of its rows' masks); entries beyond the live tile count are -1.  The tensor-core convolution (lb2_conv_desc.tile_order128)
 * deals its tiles to its persistent CTAs in this order, most expensive first, so that the cheap tiles fill the end of the launch;
 * order256 (256-row super-tiles) is not read by this build.
 * order128: cdiv(n_cap,128) ints, order256: cdiv(n_cap,256) ints, scratch: cdiv(n_cap,128) * 4 bytes. */
int lb2_tile_order(void* h, void* stream, const uint32_t* row_mask, const int32_t* row_perm, const int32_t* d_n, int32_t n_cap,
                   int32_t* order128, int32_t* order256, void* scratch);

/* Row and tile order of one offset range [k0, k1) of a kvol-27 map (0 <= k0 < k1 <= 27), for a convolution run as one launch per
 * range (lb2_conv_desc.k0 / k1).  With sub = row_mask & bits [k0, k1): perm[0..n) = the rows sorted by the stable LSD radix sort
 * of lb2_row_order on the key [sub == 0 | 2 or more bits of sub besides the centre (13) | sub without the centre bit], i.e. the rows
 * with an empty sub-mask last and the others grouped by their sub-mask; *d_live (device int32) = the number of rows with a non-empty
 * sub-mask.  No host synchronisation.  scratch >= lb2_row_order_scratch_bytes(n_cap). */
int lb2_row_order_range(void* h, void* stream, const uint32_t* row_mask, const int32_t* d_n, int32_t n_cap, int32_t k0, int32_t k1,
                        int32_t* perm, int32_t* d_live, void* scratch);

/* lb2_tile_order for a range launch: order128 over the first cdiv(*d_n, 128) tiles of perm, cost = popcount of the OR of the
 * tile's row masks restricted to [k0, k1).  Pass d_live for a range that is not the last, the map's row count for the last. */
int lb2_tile_order_range(void* h, void* stream, const uint32_t* row_mask, const int32_t* row_perm, const int32_t* d_n, int32_t n_cap,
                         int32_t k0, int32_t k1, int32_t* order128, void* scratch);

/* ---- sparse convolution  — replaces ME.MinkowskiConvolution(+Transpose) forward, with the
 * MinkowskiBatchNorm(eval)/MinkowskiReLU/residual-add/ME.cat/gate-multiply that follow it in
 * minkunet.py:13-80,431,464 fused as prologue/epilogue.
 *   out[o] = epi( sum_k [in1|in2][nbr[k][o]] @ W[k] )
 *   epi(y) = relu?( (y + pre_add[o])*scale + shift + residual[o] );  optional second output
 *   out_gated = epi(y) * gate_table[gate_idx[o]].
 * Up to two guidance passes (conditional/unconditional) share W and the map. */
typedef struct {
    const float*   in1;         /* (rows_in, c1) */
    const float*   in2;         /* (rows_in, c2) or NULL  (ME.cat as a second K segment) */
    const float*   residual;    /* (m, cout) or NULL */
    float*         out;         /* (m, cout) or NULL */
    const float*   gate_table;  /* (rows_g, cout) or NULL */
    const int32_t* gate_idx;    /* (m) or NULL (=> row 0 broadcast) */
    float*         out_gated;   /* (m, cout) or NULL */
    const float*   pre_add;     /* (m, cout) or NULL: added to the raw convolution sum before the affine
                                   (the off-centre part computed by lb2_spconv_scatter) */
    /* optional fp16 "split" companions (row = [C halfs hi | C halfs lo]; same 4C bytes as fp32):
       inputs let the tensor-core kernels gather with cp.async instead of converting in registers,
       outputs are written by the epilogue next to the fp32 tensors.  Every producer (these epilogues, lb2_gate_mul, the
       tensor-core kernels' own split of fp32 rows) writes the same split, RN = round to nearest-even, RN_sat = RN with
       results clamped to +-65504:  hi = RN_sat(x), lo = RN(x - hi).  For |x| < 131024, |x - hi - lo| <= 2^-22 |x| + 2^-25 (an
       absolute floor below |x| = 2^-3, where lo is subnormal); for larger |x| and +-inf, lo = +-inf, and NaN gives hi = lo = NaN,
       so every output that reads a non-finite (or unrepresentable) activation is non-finite, as with LB2_ALGO_FFMA. */
    const void*    in1_h;       /* (rows_in, 2*c1) fp16 or NULL */
    const void*    in2_h;       /* (rows_in, 2*c2) fp16 or NULL */
    void*          out_h;       /* (m, 2*cout) fp16 or NULL */
    void*          out_gated_h; /* (m, 2*cout) fp16 or NULL */
    /* An activation may exist as its companion only: in1/in2 may be NULL when in1_h/in2_h are given (tensor-core variants), out /
       out_gated may be NULL when out_h / out_gated_h are given, and the residual may be read from a companion (hi + lo): */
    const void*    residual_h;  /* (m, 2*cout) fp16 or NULL; used when residual == NULL */
} lb2_conv_io;

typedef struct {
    int32_t        c1, c2, cout, kvol;
    const float*   weight;      /* (kvol, c1+c2, cout) fp32 */
    const void*    weight_packed; /* tensor-core layout from lb2_pack_weights or NULL */
    const float*   scale;       /* (cout) or NULL */
    const float*   shift;       /* (cout) or NULL */
    int32_t        relu;
    const int32_t* nbr;         /* [kvol][nbr_stride] or NULL => identity map (1x1 conv) */
    int64_t        nbr_stride;
    const int32_t* d_mout;      /* device row count or NULL => mout_cap */
    int32_t        mout_cap;
    const int32_t* row_perm;    /* execution order from lb2_row_order or NULL (natural order) */
    const uint32_t* row_mask;   /* per output row: bit k set <=> nbr[k][row] >= 0 (lb2_kernel_map's row_mask) or NULL.
                                   Lets the kernels skip the index loads of absent offsets: the tensor-core kernel loads only
                                   the offsets whose bit is set, so a mask must not miss an entry of nbr */
    int32_t        npass;       /* 1 or 2 */
    lb2_conv_io    io[2];
    const int32_t* tile_order128;  /* from lb2_tile_order for this nbr / row_perm / d_mout, cdiv(mout_cap, 128) entries, or NULL (tiles
                                      in row-order sequence).  Order in which the tensor-core kernel deals its tiles to its
                                      persistent CTAs (heaviest first); ignored when nbr is NULL.  Scheduling only: results do not
                                      depend on it */
    const int32_t* tile_order256;  /* not read by this build */
    /* Offset range (tensor-core variant only): with k1 > 0 the launch runs the kernel offsets [k0, k1) of a kvol-27 map and a
       layer with one offset per accumulation group (c1 + c2 >= 176), so a conv split into ascending contiguous ranges, run as
       one launch per range, adds the same products in the same order as one launch over all 27 and gives the same bits (up to
       the sign of an exactly zero sum).  A range launch dispatches the rows row_perm[0 .. *d_mout): for a range that is not
       the last, lb2_row_order_range's live rows and d_live; for the last range, every row (d_mout = the map's row count).
       Each dispatched row starts from partial_in[pass][row] when its row_mask has a bit in [0, k0) (else from -0); a launch
       with partial_out writes its unscaled fp32 sums to partial_out[pass][row] and nothing else (no BN, residual, gate or
       outputs), a launch without it runs the epilogue.  partial_in / partial_out: (npass, mout_cap, cout) fp32, may be the same
       buffer.  row_mask is required.  k1 == 0: all offsets, partial_in / partial_out unused. */
    int32_t        k0, k1;
    const float*   partial_in;
    float*         partial_out;
} lb2_conv_desc;

#define LB2_ALGO_AUTO  0
#define LB2_ALGO_FFMA  1    /* fp32 CUDA-core implicit GEMM */
#define LB2_ALGO_TC    2    /* wgmma FP16x3 split-precision implicit GEMM (needs weight_packed), persistent CTAs over 128-row tiles */
#define LB2_ALGO_TC_TILE 3  /* the same kernel (an alias kept for callers that name it) */
int lb2_spconv_forward(void* h, void* stream, const lb2_conv_desc* d, int algo);

/* The same convolution in gather-GEMM-scatter form (what ME's GPU backend does per kernel offset) for levels
 * with few neighbours per voxel: lb2_pair_list compacts the (in,out) pairs of a kernel map per offset (optionally
 * skipping one offset, e.g. the centre 13 of a 3^3 kernel), lb2_spconv_scatter computes
 *     out[pair_out] += in[pair_in] @ W[k]        (tensor cores, FP16x3, fp32 red.add; order-dependent last bits)
 * into a buffer that lb2_spconv_forward then consumes as `pre_add` while it handles the skipped offset with
 * kvol = 1.  Cout <= 128 and packed W[k] <= 96 KB (weight-stationary). */
typedef struct {
    int32_t        c1, c2, cout, kvol;
    const void*    weight_packed;
    const int32_t* pair_in;        /* [pairs] input row  */
    const int32_t* pair_out;       /* [pairs] output row */
    const int32_t* koff;           /* [kvol+1] first pair of each offset */
    const int32_t* tile_off;       /* [kvol+1] first 128-pair tile of each offset */
    int32_t        npass;
    const float*   in1[2];
    const float*   in2[2];
    const void*    in1_h[2];       /* fp16 split companions of in1 / in2 (or NULL), see lb2_conv_io */
    const void*    in2_h[2];
    float*         out[2];         /* (m, cout) accumulation buffers */
    const int32_t* d_zero_rows;    /* rows to clear first: device count (or NULL => zero_rows_cap) */
    int32_t        zero_rows_cap;  /* 0 = caller already cleared `out` */
} lb2_scatter_desc;
size_t lb2_pair_list_scratch_bytes(void);
int lb2_pair_list(void* h, void* stream, const int32_t* nbr, int64_t nbr_stride, const int32_t* d_nout,
                  int32_t nout_cap, int32_t kvol, int32_t skip_k, int32_t* pair_in, int32_t* pair_out,
                  int32_t* koff, int32_t* tile_off, void* scratch);
int lb2_spconv_scatter_supported(int32_t c1, int32_t c2, int32_t cout, int32_t kvol);
int lb2_spconv_scatter(void* h, void* stream, const lb2_scatter_desc* d);

/* FP16 hi/lo split (power-of-two pre-scaled) + wgmma shared-memory image of a (kvol, cin, cout) fp32 weight
 * for LB2_ALGO_TC: a 256-byte header ([0] max|W| as float bits, [1] the float 2^-k), then per (k, 64-channel chunk)
 * [hi tile | lo tile], each cout rows x 128 B in the K-major SWIZZLE_128B layout, channels >= cin zero.  Values are
 * W 2^k split as hi = RN(W 2^k), lo = RN(W 2^k - hi), with k chosen so that max|W| 2^k lies in [8192, 16384), capped at
 * k = 126 (max|W| < 2^-113), k = 0 for all-zero W: any finite W gives a finite image and a finite, nonzero, normal header[1]. */
size_t lb2_packed_weight_bytes(int32_t kvol, int32_t cin, int32_t cout);
int lb2_pack_weights(void* h, void* stream, const float* weight, int32_t kvol, int32_t cin, int32_t cout,
                     void* packed);

/* Weight gradient of a sparse convolution (the backward of lb2_spconv_forward's product for one layer; the input gradient is that
 * same forward on the adjoint map with transposed weights).  For every kernel offset k
 *     dw[k] (cin x cout, fp32 row-major) = sum over o < m_out with nbr[k][o] >= 0 of x[nbr[k][o]]^T g[o]
 * x (rows_in, cin) and g (m_out, cout) fp32; nbr [kvol][nbr_stride] as lb2_spconv_forward's, or NULL (identity, kvol 1).
 * wgmma FP16x3 with the forward's split: x as an activation, g pre-scaled by a power of two 2^k (max|g| 2^k in [8192, 16384)) as a
 * weight, so the forward's error model holds with x and g in the roles of x and w (chains of 60 MMA steps, one RN add per 320 rows).
 * The rows are cut into a fixed number of chunks that depends on m_out only; each chunk's partial dw goes to scratch and a second
 * kernel adds them in chunk order: no float atomics, the same bits from run to run.
 * Shapes: kvol in {1, 8, 27}, cout in {32, 64, 96, 128, 256}, cin <= 512 and a multiple of 8 or below 8 (zero-padded); others
 * LB2_ERR_UNSUP (lb2_spconv_wgrad_scratch_bytes returns 0).  scratch >= lb2_spconv_wgrad_scratch_bytes(kvol, cin, cout, m_out). */
size_t lb2_spconv_wgrad_scratch_bytes(int32_t kvol, int32_t cin, int32_t cout, int32_t m_out);
int lb2_spconv_wgrad(void* h, void* stream, const float* x, int32_t cin, const float* g, int32_t cout, int32_t m_out,
                     const int32_t* nbr, int64_t nbr_stride, int32_t kvol, float* dw, void* scratch);

/* ---- nearest partial-scan voxel — replaces pykeops argKmin(1) in MinkUNetDiff.match_part_to_full
 * (minkunet.py:403-418): idx[q] = argmin_j |cq - ck_j|^2 over [b*2*max, x, y, z], ties -> lowest j. */
int lb2_nn_match(void* h, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                 const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, int32_t batch_scale,
                 int32_t* idx);

/* Same result as lb2_nn_match when the keys are the rows of a hash grid on a lattice of pitch key_stride
 * (the stride-16 partial-scan level): exact shell search around the query's lattice cell, exhaustive
 * fallback after max_ring shells.  Different-batch keys never match (lb2_nn_match batch_scale = 0). */
int lb2_nn_match_grid(void* h, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                      const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, lb2_grid key_grid,
                      int32_t key_stride, int32_t max_ring, int32_t* idx);

/* Variant with the key lattice in shared memory: lb2_nn_table_build re-hashes the (<= 8192) keys once per scan into
 * a compact table (`table`: lb2_nn_table_bytes() bytes), lb2_nn_match_table probes it from shared memory.  If the
 * keys do not fit the table is marked overflowing and every query takes the exhaustive path (still exact). */
size_t lb2_nn_table_bytes(void);
int lb2_nn_table_build(void* h, void* stream, const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, void* table);
int lb2_nn_match_table(void* h, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                       const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, const void* table,
                       int32_t key_stride, int32_t max_ring, int32_t* idx);

/* Variant for keys that stay fixed over many calls (the conditioning scan): lb2_nn_tree_build sorts them along a
 * Morton curve and builds a bounding-box hierarchy once (`tree`: lb2_nn_tree_bytes(nk_cap) bytes); lb2_nn_match_tree
 * searches it exactly (same result as lb2_nn_match with batch_scale = 0, incl. lowest-row ties) in ~log(nk) box
 * tests per query, independent of how far the query is from the keys.  Optional hint: hint_idx[hint_of ? hint_of[q] : q]
 * names a key row that is probably close to query q (e.g. the answer of the coarser voxel containing it; needs
 * k_coords): the search starts from that key's distance as its bound; the result does not depend on the hint. */
size_t lb2_nn_tree_bytes(int32_t nk_cap);
int lb2_nn_tree_build(void* h, void* stream, const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, void* tree);
int lb2_nn_match_tree(void* h, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                      const void* tree, int32_t nk_cap, const int32_t* k_coords, const int32_t* hint_of,
                      const int32_t* hint_idx, int32_t* idx);

/* ---- small dense layers — torch.nn.Linear (+LeakyReLU) of the gate / head MLPs
 * (minkunet.py:165-181,376-380): y = act(x @ W^T + b [+ addend]); W is (n_out, n_in) torch layout.
 * act: 0 none, 1 LeakyReLU(0.1), 2 tanh.  rows read from d_m if non-NULL.  ld_addend >= n_out when addend is given.
 * Optional input transform x' = pre_act(x + prebias[k]) (prebias (n_in) or NULL): evaluates the
 * hoisted gate MLP  latemp(cat(p,t)) = W2 . leaky(Wp.p + (Wt.t + b1)) + b2  (SURVEY.md App. D.1). */
int lb2_linear(void* h, void* stream, const float* x, int64_t ldx, const float* w, const float* b,
               const float* addend, int64_t ld_addend, int32_t m_cap, const int32_t* d_m,
               int32_t n_in, int32_t n_out, int32_t act, float* y, int64_t ldy,
               const float* prebias, int32_t pre_act);

/* The head of the U-Nets in one pass over the rows — `last` of MinkUNetDiff / MinkUNet (minkunet.py:376-380, :585-588):
 * y = out_act(W1 . LeakyReLU_0.1(W0 . x + b0) + b1), W0 (n_hid, n_in), W1 (n_out, n_hid) in torch layout; out_act as lb2_linear.
 * npass (1 or 2) row blocks x + p * x_pass_stride -> y + p * y_pass_stride (floats) share the weights and the launch.
 * n_in: multiple of 16, <= 128; n_hid <= 64; n_out <= 24; ldx a multiple of 4; x 16-byte aligned and, with npass 2,
 * x_pass_stride a multiple of 4 (rows are read with float4 loads). */
int lb2_head_mlp(void* h, void* stream, const float* x, int64_t ldx, int64_t x_pass_stride, const float* w0, const float* b0,
                 const float* w1, const float* b1, int32_t m_cap, const int32_t* d_m, int32_t n_in, int32_t n_hid,
                 int32_t n_out, int32_t out_act, int32_t npass, float* y, int64_t ldy, int64_t y_pass_stride);

/* x * w row-gather multiply (`x0*w0`, minkunet.py:431...): out[r] = x[r] * table[idx ? idx[r] : 0];
 * out_h: optional fp16 split companion of out (see lb2_conv_io); out may be NULL when out_h is given. */
int lb2_gate_mul(void* h, void* stream, const float* x, const float* table, const int32_t* idx,
                 const int32_t* d_m, int32_t m_cap, int32_t c, float* out, void* out_h);

/* out[i] = src[idx[i]]  (SparseTensor.slice / x_part.F[match], minkunet.py:418,497) */
int lb2_gather_rows(void* h, void* stream, const float* src, const int32_t* idx, int32_t n, int32_t c,
                    float* out);

/* ---- fused tail — classifier-free guidance (pipeline:153) + DPM-Solver++(2M) SDE update
 * (pipeline:162-163; diffusers DPMSolverMultistepScheduler.step) + next TensorField features and
 * coordinates (pipeline:164 -> :68-84), one thread per point coordinate.
 *   eps      = eps_u[v] + w * (eps_c[v] - eps_u[v]),  v = inverse[point]   (voxel eps, (m,3) fp32)
 *   sample   = x_t - x_init;  x0 = (sample - sigma_s*eps)/alpha_s           (fp64 like the pipeline)
 *   prev     = c_sample*sample + c_x0*x0 [+ 0.5*c_x0*(x0 - x0_prev)/r0] + c_noise*noise
 *   x_next   = fp32(x_init + prev);  coord = round_half_even(x_next / resolution)
 * coord_next is (n,4) fp32 [b, x, y, z] ready for lb2_unique_build (b from batch_col or 0).
 * x0_state (n*3 fp64) is read when second_order != 0 and always overwritten with the new x0. */
typedef struct {
    double c_sample, c_x0, c_noise, sigma_s, alpha_s, inv_r0;
    float  guidance_w, resolution;
    int32_t second_order, div_mode, f64_state;
} lb2_dpm_coef;
int lb2_guidance_dpm_step(void* h, void* stream, const float* eps_c, const float* eps_u,
                          const int32_t* inverse, const float* x_t, const double* x_init,
                          const float* noise, double* x0_state, int64_t n_points, lb2_dpm_coef coef,
                          float* eps_out, float* x_next, float* coord_next /* (n,4) */,
                          const float* batch_col /* (n) or NULL */);

/* ---- farthest point sampling — open3d farthest_point_down_sample used by preprocess_scan
 * (pipeline:97-99): start at point 0, repeatedly take the first argmax of the running min squared
 * distance (fp64).  out_idx[n_samples] selection order; dist_scratch fp64[n]. */
int lb2_farthest_point_sample(void* h, void* stream, const double* pts, int32_t n, int32_t n_samples,
                              int32_t* out_idx, double* dist_scratch);

/* Batched farthest point sampling: n_scans ragged scans, scan b = pts rows [d_offsets[b], d_offsets[b+1]) (d_offsets: device
 * int64[n_scans+1]), max_n >= every scan's size, n_samples <= every scan's size.  out_idx (n_scans, n_samples) int32 holds each
 * scan's selection order in scan-local indices, bit-identical to lb2_farthest_point_sample on that scan.  One thread-block
 * cluster per scan with the scan's coordinates in shared memory, so the scans run concurrently; a scan may have at most
 * lb2_fps_batched_capacity(h) points (0: the device cannot run the cluster). */
int64_t lb2_fps_batched_capacity(void* h);
int lb2_farthest_point_sample_batched(void* h, void* stream, const double* pts, const int64_t* d_offsets, int32_t n_scans,
                                      int32_t max_n, int32_t n_samples, int32_t* out_idx);

/* ---- evaluation metrics — lidiff/utils/metrics.py:63-221, histogram_metrics.py:7-51, eval_path.py:65-170.
 * Points are fp64 rows (n, 3).  Every result is deterministic: integer counts, fp64 sums in a fixed order. */

/* Exact 1-NN point-to-cloud distance — replaces open3d PointCloud.compute_point_cloud_distance (KDTreeFlann 1-NN in fp64;
 * metrics.py:70,131-132,153-156).  lb2_pc_tree_build sorts the reference cloud along a Morton curve and builds a box hierarchy
 * over it (`tree`: lb2_pc_tree_bytes(n) bytes, n >= 1); lb2_pc_nn gives, for every query, dist[q] = sqrt(dx^2 + dy^2 + dz^2)
 * (fp64, no FMA contraction) to its nearest reference point and, if idx != NULL, idx[q] = that point's index (lowest index on
 * equal distances).  ~log(n) box tests per query, however far the query is from the cloud.  Rows with a NaN or infinite
 * coordinate do not affect the tree's shape or the search cost: they are left out of its bounding box and node boxes and sorted
 * after every finite row (a finite outlier still coarsens the Morton grid; the results stay exact).  Only a finite squared distance
 * counts: a query with a NaN or infinite coordinate does not search, reference points with one are nobody's neighbour, and a query
 * without a finite squared distance to any point (those, a reference without a finite point, or one whose squared distances all
 * overflow) gets idx[q] = -1 and dist[q] = +inf.  The results are exact for finite coordinates whose squared distances do not
 * overflow; non-finite ones never fault.  scratch >= lb2_pc_nn_scratch_bytes(nq). */
size_t lb2_pc_tree_bytes(int32_t n_cap);
size_t lb2_pc_nn_scratch_bytes(int32_t nq_cap);
int lb2_pc_tree_build(void* h, void* stream, const double* pts, int32_t n, void* tree);
int lb2_pc_nn(void* h, void* stream, const double* q, int32_t nq, const void* tree, double* dist, int32_t* idx, void* scratch);

/* Deterministic segmented sum (the backward of a row gather, e.g. the Chamfer loss' x[idx]):
 *     out[s][j] = sum over i in [offsets[s], offsets[s + 1]) of values[order[i]][j], added in ascending i
 * values (rows, c) fp32, or fp64 with f64 = 1; order int64 (NULL = identity); offsets int64[nseg + 1]; out (nseg, c). */
int lb2_segment_sum(void* h, void* stream, const void* values, int32_t f64, const int64_t* order, const int64_t* offsets,
                    int64_t nseg, int32_t c, void* out);

/* Deterministic segmented product-sum under skewed segment lengths (the gradient of the conditioning gates' gather x * table[idx]):
 *     out[s][j] = sum over i in [offsets[s], offsets[s + 1]) of a[order[i]][j] * b[order[i]][j]        (b == NULL: of a[order[i]][j])
 * a, b (rows, c) fp32, 1 <= c <= 256 (others: LB2_ERR_ARG); order int64[nrows] (NULL = identity); offsets int64[nseg + 1],
 * non-decreasing with offsets[0] = 0 and offsets[nseg] = nrows; out (nseg, c) fp32; scratch >= lb2_segment_dot_scratch_bytes(nrows, c).
 * nseg == 0 writes nothing; nrows == 0 writes zeros.  The work is split by position, not by segment, so one segment that holds
 * every row costs what many short ones do.  Summation order, per channel j, with R = LB2_SEGMENT_DOT_R, every product one
 * round-to-nearest multiply and every addition one round-to-nearest add (no FMA):
 *   - chunk k is the positions [k R, min((k + 1) R, nrows)); the pieces of segment s are its non-empty intersections with the chunks;
 *   - a piece's sum starts from +0 and adds its products in ascending position i;
 *   - a segment with one piece is that piece's sum; a segment with several is +0 plus its pieces' sums in ascending chunk order; a
 *     segment without rows is +0.
 * So the result depends on the inputs only (no atomics), and a NaN or inf in a row reaches its own segment's sum and no other. */
#define LB2_SEGMENT_DOT_R 128
size_t lb2_segment_dot_scratch_bytes(int64_t nrows, int32_t c);
int lb2_segment_dot(void* h, void* stream, const float* a, const float* b, const int64_t* order, const int64_t* offsets,
                    int64_t nrows, int64_t nseg, int32_t c, float* out, void* scratch);

/* Synchronised batch norm (training mode over the rows of every rank; lidiff_b200.me.MinkowskiSyncBatchNorm).  Each rank passes its
 * own rows x (n, c) fp32, 0 <= n < 2^31, 1 <= c <= 1024; the caller combines the int64 word arrays across ranks between the calls
 * (MAX for *max_words, SUM for *sum_words / sq_words) and the global row count N = sum of n must stay below 2^31 (a combined
 * count outside 1 <= N < 2^31 makes mean, var, invstd, y, dx and the running statistics NaN, as the words may have wrapped).  Every output
 * depends only on the multiset of rows: not on their order, the launch or the split across ranks.  Per channel j, with
 * RN64 / RN32 one round-to-nearest-even fp64 / fp32 operation each (no FMA), e(v) the exponent with v < 2^e(v) (e(0) = 0) and
 * RNI(v) the nearest integer (ties to even):
 *
 *   lb2_sync_bn_max      max_words[2j] = bits of M = the largest finite |x|, max_words[2j+1] = 1 if x holds a NaN or +-inf.  [MAX]
 *   lb2_sync_bn_sum      q = RNI(x 2^s), s = 62 - e(M), |q| <= 2^62; sum_words[2j] = sum (q >> 32), sum_words[2j+1] = sum (q & (2^32 - 1)),
 *                        sum_words[2c] = n.  S = sum_words[2j] 2^32 + sum_words[2j+1] is exact.                              [SUM]
 *   lb2_sync_bn_sumsq    mean[j] = mu = RN64(S / N) 2^-s (the quotient of the integers rounded once); then d = RN64(x - mu),
 *                        p = RNI(d 2^t), t = 62 - e(RN64(M + |mu|)), and sq_words[4j + k] = the sum of 32-bit limb k of p^2 (< 2^125).
 *                        T = sum_k sq_words[4j + k] 2^(32 k) is exact.                                                       [SUM]
 *   lb2_sync_bn_apply    var[j] = RN64(T / N) 2^-2t (biased, as torch normalises), invstd[j] = RN64(1 / RN64(sqrt(RN64(var + eps)))),
 *                        y = RN32(RN64(RN64(RN64(d invstd) gamma) + beta)) (gamma / beta NULL: 1 / 0);
 *                        with running statistics (a = momentum): rm = RN32(RN64(RN64((1 - a) rm) + RN64(a mu))),
 *                        rv = RN32(RN64(RN64((1 - a) rv) + RN64(a u))), u = RN64(RN64(var N) / (N - 1)) (N = 1: NaN).
 * A flagged channel (max_words[2j+1]) has mu = var = invstd = NaN and y[:, j] = NaN on every rank; the other channels keep their bits.
 *
 * Words: |q|, |p| <= 2^62 give 32-bit limbs, and N < 2^31 rows keep every word's sum below 2^63 on one rank and after the SUM across
 * ranks.  Error against exact arithmetic (m, v the exact mean and biased variance of the union, B = M + |mu| <= 2M (1 + 2^-52)):
 *   |mu - m|   <= 2^-62 M + 2^-53 |m|
 *   |var - v|  <= 2^-50 v + 2^-59 B sqrt(v) + 2^-100 B^2
 * (each q and p is within 1/2 of its scaled value, d carries one fp64 rounding, the quotients one each).  For v >= 2^-40 M^2 the
 * relative error of var is below 2^-37, far below fp32's 2^-24.
 *
 * Backward, with xhat = RN64(d invstd) and g = RN64(dy xhat) in the forward's formulas:
 *   lb2_sync_bn_backward_max   max_words[3j] = bits of the largest finite |dy| (fp32), [3j+1] = bits of the largest finite |g| (fp64),
 *                              [3j+2] = 1 if a dy or g is NaN or +-inf.                                                      [MAX]
 *   lb2_sync_bn_backward_sum   a = RNI(dy 2^sa), sa = 62 - e(max|dy|); b = RNI(g 2^sb), sb = 62 - e(max|g|); sum_words[4j .. 4j+3] =
 *                              the hi / lo words of sum a and of sum b as above.  This rank's parameter gradients (NULL: skipped)
 *                              dbeta = RN32(RN64(A) 2^-sa), dgamma = RN32(RN64(Bs) 2^-sb) from these local words.            [SUM]
 *   lb2_sync_bn_backward_apply mdy = RN64(A / N) 2^-sa, mg = RN64(Bs / N) 2^-sb from the combined words, N = *count (the forward's
 *                              sum_words[2c]); dx = RN32(RN64(k RN64(RN64(dy - mdy) - RN64(xhat mg)))), k = RN64(gamma invstd).
 * A flagged channel has dx[:, j], dgamma[j], dbeta[j] = NaN.  No float atomics. */
int lb2_sync_bn_max(void* h, void* stream, const float* x, int64_t n, int32_t c, int64_t* max_words);
int lb2_sync_bn_sum(void* h, void* stream, const float* x, int64_t n, int32_t c, const int64_t* max_words, int64_t* sum_words);
int lb2_sync_bn_sumsq(void* h, void* stream, const float* x, int64_t n, int32_t c, const int64_t* max_words, const int64_t* sum_words,
                      double* mean, int64_t* sq_words);
int lb2_sync_bn_apply(void* h, void* stream, const float* x, int64_t n, int32_t c, const int64_t* max_words, const int64_t* sum_words,
                      const double* mean, const int64_t* sq_words, const float* gamma, const float* beta, double eps, double momentum,
                      float* running_mean, float* running_var, double* var, double* invstd, float* y);
int lb2_sync_bn_backward_max(void* h, void* stream, const float* dy, const float* x, int64_t n, int32_t c, const double* mean,
                             const double* invstd, int64_t* max_words);
int lb2_sync_bn_backward_sum(void* h, void* stream, const float* dy, const float* x, int64_t n, int32_t c, const double* mean,
                             const double* invstd, const int64_t* max_words, int64_t* sum_words, float* dgamma, float* dbeta);
int lb2_sync_bn_backward_apply(void* h, void* stream, const float* dy, const float* x, int64_t n, int32_t c, const double* mean,
                               const double* invstd, const float* gamma, const int64_t* max_words, const int64_t* sum_words,
                               const int64_t* count, float* dx);

/* Point normals as open3d 0.17's PointCloud.estimate_normals() computes them (KDTreeSearchParamKNN(30), fast_normal_computation;
 * tools/diff_completion_pipeline.py:204-212), in two steps over a tree from lb2_pc_tree_build(pts, n):
 *   lb2_pc_knn      exact self-k-nearest neighbours, 1 <= k <= 32 (larger k: LB2_ERR_UNSUP).  With k_eff = min(k, n), row j of
 *                   idx (int32[n][k_eff]) lists the k_eff points nearest to point j, itself included, ordered by
 *                   (d², index) with d² = (dx*dx + dy*dy) + dz*dz in fp64 (no FMA contraction, as lb2_pc_nn); ties go to the
 *                   lower index.  d2 (double[n][k_eff]) receives the distances if not NULL.  n must be the tree's point count;
 *                   if it is not, every row is written empty.  An empty slot holds index -1 and d² = +inf: the slots of a point
 *                   with a NaN or infinite coordinate, and those past the number of finite points (the neighbours are exact for
 *                   finite coordinates whose squared distances do not overflow; non-finite ones never fault).
 *   lb2_pc_normals  normals[i] (double[n][3]) = FastEigen3x3 of the one-pass cumulant covariance of the k neighbours idx[i][0..k)
 *                   (idx: int32[n][k], k = the k_eff of lb2_pc_knn): sums of x, y, z, xx, xy, xz, yy, yz, zz in neighbour order,
 *                   divided by k, C = E[pp^T] - E[p]E[p]^T (the identity when k < 3); the eigenvector of the smallest eigenvalue,
 *                   unoriented, (0, 0, 1) where the solver gives the zero vector or C has a NaN or infinite entry (the
 *                   cumulants overflow once a neighbourhood's coordinates pass ~1e154), NaN where the row holds an index outside
 *                   [0, n) (an empty lb2_pc_knn slot; nothing is read for it).  Every operation is rounded on its own, so C is
 *                   bit-exact against a sequential host evaluation and the normal differs from one only through acos / cos. */
int lb2_pc_knn(void* h, void* stream, const void* tree, int32_t n, int32_t k, int32_t* idx, double* d2);
int lb2_pc_normals(void* h, void* stream, const double* pts, int32_t n, const int32_t* idx, int32_t k, double* normals);

/* np.histogramdd(pts, bins, range=[-50, 50]^3) binning (metrics.py:93-101, histogram_metrics.py:11): per axis
 * bin = searchsorted(edges, x, 'right') - 1 with edges (bins + 1 fp64, np.linspace of the range) from the caller, a value equal
 * to the last edge in the last bin, points outside the range on any axis dropped.  Outputs (each optional, cleared first):
 * bits = occupancy bitset of bins^3 bits in C order (x slowest, z fastest; bit c at word c / 32, bit c % 32), counts = uint32
 * per cell (bins^3), n_in = number of points inside the range.  bins <= 2048. */
int lb2_voxel_occupancy(void* h, void* stream, const double* pts, int32_t n, const double* edges, int32_t bins,
                        uint32_t* bits, uint32_t* counts, uint64_t* n_in);

/* CompletionIoU confusion counts (metrics.py:103-105) of two occupancies of nbits cells:
 * out[0] = tp = |gt & pred|, out[1] = fn = |gt & ~pred|, out[2] = fp = |~gt & pred|. */
int lb2_occupancy_confusion(void* h, void* stream, const uint32_t* bits_gt, const uint32_t* bits_pred, int64_t nbits, uint64_t* out);

/* BEV histogram of histogram_metrics.py:13,16 (counts clipped to 1, summed over z) from an occupancy of bins^3 cells:
 * bev[x * bins + y] = number of occupied z cells of column (x, y). */
int lb2_occupancy_bev(void* h, void* stream, const uint32_t* bits, int32_t bins, uint32_t* bev);

/* Jensen-Shannon distance of two count histograms as histogram_metrics.py:15-44 computes it (normalise each by its sum, then
 * scipy.spatial.distance.jensenshannon, natural log): *out = sqrt((sum rel_entr(p, m) + sum rel_entr(q, m)) / 2), m = (p + q) / 2;
 * NaN if either histogram is empty.  scratch >= lb2_jsd_scratch_bytes(n). */
size_t lb2_jsd_scratch_bytes(int64_t n);
int lb2_jsd(void* h, void* stream, const uint32_t* hist_a, const uint32_t* hist_b, int64_t n, double* out, void* scratch);

/* Per-direction distance statistics (RMSE / Chamfer means, metrics.py:72,134; precision / recall counts, metrics.py:158-165):
 * *sum_out = fp64 sum of the n distances; counts_out[k] = number of distances < thresholds[k] (NaN and +inf distances are never
 * counted).  The thresholds must be ascending and not NaN (each distance is binary-searched among them; other orders give wrong
 * counts without an error), nt <= 4096.  Summation order, with nblk = max(1, min(ceil(n / 256), 1024)) and every addition one
 * round-to-nearest fp64 add: thread t of block b sums the elements b 256 + t + k nblk 256 in increasing k from +0; each block
 * reduces its 256 sums by the tree s[t] += s[t + o], o = 128, 64, ..., 1; the block sums are added from +0 in block order.
 * scratch >= lb2_dist_stats_scratch_bytes(nt). */
size_t lb2_dist_stats_scratch_bytes(int32_t nt);
int lb2_dist_stats(void* h, void* stream, const double* dist, int32_t n, const double* thresholds, int32_t nt,
                   double* sum_out, uint64_t* counts_out, void* scratch);

/* ---- ground-truth maps — lidiff/map_from_scans.py:63-96 (the static map `<seq>/map_clean.npy` that the evaluation and the
 * reference's dataloader read).  The reference appends every filtered, transformed scan to the map and de-duplicates the whole map
 * again; since an existing map point always precedes a new scan in that concatenation, the result equals one global
 * first-occurrence de-duplication over all scans, which these calls build scan by scan with a persistent table.
 *
 * The table is an lb2_grid used as a set of voxel keys: keys uint64[cap], vals int32[2 * cap] = [0, cap) claim (lowest point index
 * of the call that created the slot), [cap, 2 cap) map row (-1 until the creating call has finished).  Key packing: 3 x 21 bit
 * biased signed voxel indices (no batch field), i.e. +-2^20 voxels per axis (+-104 km at 0.1 m). */
#define LB2_MAP_AXIS_BITS 21
typedef struct { float m[12]; } lb2_pose;   /* rows 0..2 of the 4x4 scan-to-map pose, row-major, fp32 */

/* lb2_map_rehash clears `table` (cap a power of two) and inserts the (key, row) pairs of old_table (keys NULL / cap 0: none), so a
 * new table is made with old_table empty and a full one is grown into a larger one.  old_table.cap_table <= table.cap_table. */
int lb2_map_rehash(void* h, void* stream, lb2_grid old_table, lb2_grid table);

/* One scan: `points` (n, 4) fp32 rows x, y, z, remission; `labels` uint32[n] or NULL (no label filter).
 *   keep     (l & 0xFFFF) in (1, 252)  and  sqrt_rn(((x^2 + y^2) + z^2) + r^2) > 3.5      (map_from_scans.py:74-85)
 *   p'_k     ((m[4k] x + m[4k+1] y) + m[4k+2] z) + m[4k+3]  in fp32, every operation rounded (no FMA)   (:87-88, w = 1)
 *   voxel    floor(p' / voxel_size): div_mode 0 true fp32 division (the reference's --cpu run), 1 multiply by fp32(1 / voxel_size)
 *            (PyTorch's CUDA scalar division, its default device)
 * A kept point whose voxel already has a map row is dropped; among the points of this call that share a new voxel the lowest index
 * wins, and the winners are appended in point order as fp32 p' rows map[map_n ...].  d_out (device int32[2]): [0] = number of new
 * rows, [1] = status, bit0 = a kept point's voxel index is outside the key range (that point is not inserted; the map is then
 * incomplete and the caller should treat the build as failed).  n <= 4M; cap_table >= 2 * (map_n + n); map_cap >= map_n + n.
 * Per-call work is O(n): nothing is cleared per call.  scratch >= lb2_map_scan_scratch_bytes(n). */
size_t lb2_map_scan_scratch_bytes(int32_t n_cap);
int lb2_map_scan(void* h, void* stream, const float* points, const uint32_t* labels, int32_t n, lb2_pose pose, float voxel_size,
                 int32_t div_mode, lb2_grid table, float* map, int32_t map_n, int32_t map_cap, int32_t* d_out, void* scratch);

/* ---- training / test samples — lidiff/datasets/dataloader/SemanticKITTITemporal.py:82-105 and lidiff/utils/collations.py:44-51
 * (TemporalKITTISet.__getitem__ before the farthest point sampling).  Both calls are order-preserving compactions: the kept rows
 * are written as fp64 (x, y, z) rows in input order, *d_count (device int32) = their number.  Inputs of up to 2^31 - 1 rows. */

/* lb2_select_points: row i of `points` (n rows of `stride` = 3 or 4 values, fp32 or fp64 (fp64 != 0); only x, y, z are read) is kept
 * when every test below holds, in this order (each later test sees the row as the earlier steps left it):
 *   finite   x, y and z are finite (numpy's comparisons with NaN are false)
 *   labels   (uint32[n] or NULL)  1 < (l & 0xFFFF) < 252                                           (:86-91)
 *   range    r_min < d < r_max, d = |p - center| in the input frame:
 *              LB2_RANGE_FP32   fp32: sqrt_rn((dx*dx + dy*dy) + dz*dz), dx = fp32(x) - fp32(center.x), bounds rounded to fp32
 *                               (the scan: a float32 array and numpy's float32 sum, :92-93)
 *              LB2_RANGE_FP64   the same in fp64 (the map crop about the pose translation, :100-102)
 *   transform (has_transform)  p'_k = ((m[4k] x + m[4k+1] y) + m[4k+2] z) + m[4k+3] in fp64 (the map into the scan frame, :103-104)
 *   height   (has_z_min)  p'.z > z_min in fp64                                                          (:94, :105)
 * Every operation is rounded on its own (no FMA contraction), so each decision is the one numpy takes on the same values.
 * scratch >= lb2_select_points_scratch_bytes(n). */
#define LB2_RANGE_NONE 0
#define LB2_RANGE_FP32 1
#define LB2_RANGE_FP64 2
typedef struct {
    int32_t range_mode;
    double  center[3];
    double  r_min, r_max;
    int32_t has_transform;
    double  transform[12];      /* rows 0..2 of a 4x4, row-major */
    int32_t has_z_min;
    double  z_min;
} lb2_select_desc;
size_t lb2_select_points_scratch_bytes(int64_t n);
int lb2_select_points(void* h, void* stream, const void* points, int32_t fp64, int64_t n, int32_t stride, const uint32_t* labels,
                      const lb2_select_desc* desc, double* out, int32_t* d_count, void* scratch);

/* lb2_viewpoint_filter: o3d VoxelGrid.create_from_point_cloud(part, voxel_size).check_if_included(full) with the semantics of the
 * open3d shim (lidiff_b200/shims/open3d/geometry.py): origin = per-axis minimum of `part` - voxel_size / 2, cell of p =
 * floor((p - origin) / voxel_size) in fp64; row i of `full` (fp64 (n_full, 3)) is kept iff its cell holds a row of `part` (fp64
 * (n_part, 3), finite).  Cell indices are keyed in [0, 2^21) per axis; a `full` row outside that range is not included, a `part` row
 * outside it sets status bit 0 (the result is then incomplete).  d_out (device int32[2]): [0] = kept rows, [1] = status.
 * An empty `part` includes nothing.  scratch >= lb2_viewpoint_filter_scratch_bytes(n_part, n_full). */
size_t lb2_viewpoint_filter_scratch_bytes(int32_t n_part, int64_t n_full);
int lb2_viewpoint_filter(void* h, void* stream, const double* part, int32_t n_part, const double* full, int64_t n_full,
                         double voxel_size, double* out, int32_t* d_out, void* scratch);

/* ---- refinement samples — lidiff/utils/pcd_preprocess.py:78-129 (aggregate_pcds) and
 * lidiff/datasets/dataloader/SemanticKITTITemporalAggr.py:69-99 (TemporalKITTISet.__getitem__).  Order-preserving compactions like
 * the two calls above: kept rows are written as fp64 (x, y, z) rows in input order.  Inputs of up to 2^31 - 1 rows, addressed with
 * 64-bit indices; every operation is rounded on its own (no FMA contraction), in the order given. */

/* lb2_aggregate_window: the scans of one window, concatenated: `points` (n, 4) fp32 rows x, y, z, remission and `labels` uint32[n].
 * segments[nseg] (device) = the first row of every scan, ascending (segments[0].start = 0; empty scans share a start) and rows 0..2
 * of its fp64 scan-to-world pose; undo (host, 12 fp64) = rows 0..2 of inv(pose of the window's frame).  Row i is kept when
 *   labels   (l & 0xFFFF) < 252                    (classes 0 and 1 are kept)
 *   range    sqrt_rn((x*x + y*y) + z*z) > 3.5 in fp32 over x, y, z       (NaN fails, +-inf passes)
 * and written as undo(pose(p)), each p'_k = ((m[4k] x + m[4k+1] y) + m[4k+2] z) + m[4k+3] in fp64 (numpy's apply_transform).
 * d_out (device int32[2]): [0] = kept rows, [1] = kept rows of [0, split) (the split between pcd_full and pcd_part when the frame
 * scan is uploaded last and starts at `split`).  scratch >= lb2_aggregate_window_scratch_bytes(n). */
typedef struct {
    int64_t start;
    double  m[12];
} lb2_segment;
size_t lb2_aggregate_window_scratch_bytes(int64_t n);
int lb2_aggregate_window(void* h, void* stream, const float* points, const uint32_t* labels, int64_t n, const lb2_segment* segments,
                         int32_t nseg, const double* undo, int64_t split, double* out, int32_t* d_out, void* scratch);

/* lb2_jitter_filter: jitter_point_cloud (pcd_transforms.py:35-40) and the 50 m test of the noisy rows.  points, randn fp64 (n, 3);
 * randn is numpy's standard normal draw.  w = clip(sigma * r, -clip, clip) + p per coordinate (clip: fmin(fmax(v, -clip), clip)),
 * kept where sqrt_rn((x*x + y*y) + z*z) < max_range in fp64.  *d_count (device int32) = kept rows.
 * scratch >= lb2_jitter_filter_scratch_bytes(n). */
size_t lb2_jitter_filter_scratch_bytes(int64_t n);
int lb2_jitter_filter(void* h, void* stream, const double* points, const double* randn, int64_t n, double sigma, double clip,
                      double max_range, double* out, int32_t* d_count, void* scratch);

/* lb2_voxel_first_f64: ME.utils.sparse_quantize(p / voxel_size, return_index=True) on fp64 (n, 3) rows, then the max_range test:
 * the voxel of a row is floor(p / voxel_size) per axis (the true fp64 quotient), packed as the map keys above (+-2^20 voxels per
 * axis); the lowest row index of every voxel wins, and a winner is kept where sqrt_rn((x*x + y*y) + z*z) < max_range in fp64.
 * Rows with a NaN / inf coordinate are never kept.  One-shot table of the next power of two >= 2n slots.  d_out (device int32[2]):
 * [0] = kept rows, [1] = status, bit0 = a finite row's voxel index is outside the key range (the result is then incomplete).
 * scratch >= lb2_voxel_first_f64_scratch_bytes(n). */
size_t lb2_voxel_first_f64_scratch_bytes(int64_t n);
int lb2_voxel_first_f64(void* h, void* stream, const double* points, int64_t n, double voxel_size, double max_range, double* out,
                        int32_t* d_out, void* scratch);

/* ---- host random streams drawn on the device (rng.cu, lidiff_b200/rng.py) ------------------------------------------------------
 *
 * lb2_mt19937_words: the next n tempered MT19937 words of the 624-word state `state` (device uint32[624], updated in place) at
 * position pos in [0, 624] (numpy's pos; torch's 625 - left; 624 = twist before the next word) -> out (device uint32[n]);
 * *pos_out (host) = the position afterwards.  One CTA; the twist is the reference MT19937's, word for word.
 *
 * lb2_legacy_gauss: numpy's legacy_gauss (the polar method of RandomState.randn) called n_out times over `words` (device, 16-byte
 * aligned, from lb2_mt19937_words; n_words / 4 attempts) with the incoming cache (has_gauss, gauss) -> out (device fp64[n_out]).
 * Attempt k reads words 4k .. 4k+3: x = 2 ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 - 1 for x1 then x2, r2 = x1 x1 + x2 x2 (no FMA),
 * rejected when r2 >= 1 or r2 == 0; f = sqrt(-2 log(r2) / r2); outputs f x2, then f x1.  log is glibc's: where the double-double
 * log of r2 lies more than `band` ulp from a rounding midpoint its leading word is used (glibc's log errs by less than 0.519 ulp,
 * so it returns the correct rounding there); the other attempts are copied to the host and resolved with libm's log.
 * band in [0, 0.5] (LB2_GAUSS_BAND by default; 0.5 resolves every attempt on the host).  The call synchronises `stream` (one read
 * of the attempt and deferred counts, one of the deferred attempts).  *info (host): words_used = the words numpy consumed,
 * deferred = attempts resolved on the host, (has_gauss, gauss) = numpy's cache afterwards; short_words = 1 when the words held
 * too few accepted attempts: nothing is valid then, call again with more words of the same stream.
 * scratch >= lb2_legacy_gauss_scratch_bytes(n_words, n_out).
 *
 * lb2_randperm: torch.randperm(n) of the CPU generator: out (device int64[n]) = the identity shuffled by z_i = words[i] % (n - i),
 * swap(out[i], out[i + z_i]) for i < n - 1 in order (words: device uint32[n - 1] from lb2_mt19937_words), computed in rounds of
 * deterministic reservations by one cooperative grid.  n < LB2_RANDPERM_MAX_N (torch draws 64-bit words from there: LB2_ERR_ARG).
 * *d_rounds (device int32, may be NULL) = the reservation rounds.  scratch >= lb2_randperm_scratch_bytes(n). */
#define LB2_GAUSS_BAND (1.0 / 32.0)
#define LB2_RANDPERM_MAX_N 214748364LL      /* UINT32_MAX / 20 */
typedef struct {
    int64_t words_used;
    int64_t deferred;
    int32_t short_words;
    int32_t has_gauss;
    double  gauss;
} Lb2GaussInfo;
int lb2_mt19937_words(void* h, void* stream, uint32_t* state, int32_t pos, int64_t n, uint32_t* out, int32_t* pos_out);
size_t lb2_legacy_gauss_scratch_bytes(int64_t n_words, int64_t n_out);
int lb2_legacy_gauss(void* h, void* stream, const uint32_t* words, int64_t n_words, int64_t n_out, int32_t has_gauss, double gauss,
                     double band, double* out, Lb2GaussInfo* info, void* scratch);
size_t lb2_randperm_scratch_bytes(int64_t n);
int lb2_randperm(void* h, void* stream, const uint32_t* words, int64_t n, int64_t* out, int32_t* d_rounds, void* scratch);

/* ---- point-cloud images without a display (render.cu, lidiff_b200/render.py) — the view of lidiff/vis_pcd.py's
 * o3d.visualization.draw_geometries as an 8-bit RGB image.  Every fp64 operation below is rounded on its own (no FMA contraction)
 * and dot products are summed left to right, a.b = (a.x b.x + a.y b.y) + a.z b.z, so a sequential host evaluation gives the same keys
 * and colours bit for bit.  Both calls are deterministic and use no float atomics.
 *
 * Camera (lb2_render_camera; the caller computes every transcendental): F = normalize(front), right = normalize(up x F),
 * up' = normalize(F x right), eye = lookat + F distance, with normalize(a) = a / sqrt(a.a) per component and
 * a x b = (a.y b.z - a.z b.y, a.z b.x - a.x b.z, a.x b.y - a.y b.x).  focal = (height / 2) / tan(fov / 2) in pixels.
 *
 * lb2_render_splat: for point p (fp64 (n, 3), n < 2^32 - 1) with d = p - eye:
 *   depth = -(d.F),  u = width / 2 + (focal (d.right)) / depth,  v = height / 2 - (focal (d.up')) / depth.
 * Skipped: a NaN / inf coordinate, depth <= 1e-3 distance (no far plane), a NaN u or v.  With a = u - s/2, b = u + s/2 (s = point_size,
 * each rounded), each clamped to [-1, width + 1], the point covers the columns c in [0, width) with a <= c + 0.5 < b, i.e.
 * ceil(a - 0.5) <= c < ceil(b - 0.5); rows likewise from v and height.  An integer s therefore covers s x s pixels, as an OpenGL square
 * point of that size does.  Each covered pixel takes atomicMin(keys[row width + col], (float_bits(float(depth)) << 32) | index): the
 * nearest point wins and ties go to the lower index, whatever the launch order.  keys (device uint64[height width]) must be filled
 * with LB2_KEY_EMPTY (background) by the caller; several splats may accumulate into one buffer.  0 < point_size <= 4096.
 *
 * lb2_render_shade: rgb (device uint8[height][width][3]) from the keys.  Background: (255, 255, 255).  Otherwise, with i = the key's
 * index: the base colour c is float(colors[i]) (colors fp64 (n, 3), NULL: none) or open3d's ColorMapJet of
 * t = (z_i - z_lo) / (z_hi - z_lo) clamped to [0, 1] (t = 0 when z_hi == z_lo): c = (jet(2t - 1.5), jet(2t - 1.0), jet(2t - 0.5)) in fp64 with
 *   jet(x) = 0 (x <= -0.75), ((x + 0.75) / 0.5) 1 + 0 (x <= -0.25), 1 (x <= 0.25), ((x - 0.25) / 0.5) (-1) + 1 (x <= 0.75), else 0,
 * each channel rounded to fp32.  With normals (fp64 (n, 3), NULL: none) the two-sided headlight factor
 * k = 0.25f + 0.75f |float(n_i.F)| in fp32 (k = 1 when float(n_i.F) is not finite), else k = 1.  Each channel:
 * rint(255f clamp(c k, 0, 1)) in fp32, round half to even, where clamp maps NaN to 0.  A point whose pixels are all covered by
 * nearer points is never read. */
typedef struct {
    double  lookat[3];
    double  front[3];       /* from the look-at point towards the eye; need not be unit length, must not be zero */
    double  up[3];
    double  distance;       /* > 0 */
    double  focal;          /* > 0, pixels */
    int32_t width, height;  /* > 0 */
} lb2_render_camera;
int lb2_render_splat(void* h, void* stream, const double* pts, int64_t n, const lb2_render_camera* cam, double point_size,
                     uint64_t* keys);
int lb2_render_shade(void* h, void* stream, const uint64_t* keys, const double* pts, const double* normals, const double* colors,
                     double z_lo, double z_hi, const lb2_render_camera* cam, uint8_t* rgb);

/* ---- uniform surface sampling of triangle meshes (mesh.cu, lidiff_b200/mesh.py) — open3d 0.17's
 * TriangleMesh::SamplePointsUniformly under libstdc++, which lidiff/utils/metrics.py:37 (Metrics3D.convert_to_pcd) calls with
 * 1 000 000 points.  Every fp64 operation below is rounded on its own (no FMA contraction) so that a sequential host evaluation
 * (tests/mesh_reference.py) gives the same bits.  Deterministic; no float atomics.
 *
 * Inputs: verts fp64 (n_verts, 3), tris int32 (n_tris, 3), N = n_points.
 *   area_t = 0.5 |x × y| with x = p0 - p1, y = p0 - p2 (p_k = verts[tris[t][k]]), a × b as in lb2_render_*, and
 *     |c| = sqrt((c0 c0 + c1 c1) + c2 c2);
 *   S = area_0 + area_1 + ... left to right (surface_area += area);
 *   cdf_0 = area_0 / S, cdf_t = area_t / S + cdf_{t-1}: a sequential chain (the quotients are independent, the adds are not);
 *   n_t = round(cdf_t N), half away from zero; triangle t owns the points [n_{t-1}, n_t) (n_{-1} = 0), so point i lies on the
 *     first t with n_t > i.
 * Random numbers: point i reads words[4i .. 4i+3] (one uint4; words from lb2_mt19937_words, so a call consumes exactly 4N words of
 * the stream): r1 from (words[4i], words[4i+1]), r2 from (words[4i+2], words[4i+3]), each libstdc++'s
 * generate_canonical<double, 53> of std::mt19937 (uniform_real_distribution<double>(0, 1)):
 *   r = RN(w_lo + w_hi 2^32) 2^-64, and r = nextafter(1, 0) when r >= 1.
 * The point: s = sqrt(r1), a = 1 - s, b = s (1 - r2), c = s r2; per axis p = (a v0 + b v1) + c v2.
 *
 * lb2_mesh_sample_prepare: the areas (area: device fp64[n_tris]), S and the n_t (kept in scratch) and *d_info (device).  Bad input
 * found on the device is reported in d_info->status, never by a fault:
 *   LB2_MESH_BAD_INDEX     a vertex index outside [0, n_verts) (that triangle's area is 0);
 *   LB2_MESH_NON_FINITE    a triangle uses a vertex with a NaN / inf coordinate;
 *   LB2_MESH_BAD_AREA      S is 0, or not finite (n_t are then not computed);
 *   LB2_MESH_BAD_COUNT     the last n_t is not N (cannot happen while n_tris N < 2^51: the chain's rounding stays below 1/2).
 * A caller reads *d_info once and calls lb2_mesh_sample_points only when status == 0.  n_points in [1, 2^53), n_tris >= 1,
 * n_verts >= 1.  scratch >= lb2_mesh_sample_scratch_bytes(n_tris), 16-byte aligned.
 * lb2_mesh_sample_points: out (device fp64 (n_points, 3)) from the n_t of the prepare call on the same verts / tris / n_points / scratch;
 * words: device uint32[4 n_points], 16-byte aligned. */
#define LB2_MESH_BAD_INDEX   1
#define LB2_MESH_NON_FINITE  2
#define LB2_MESH_BAD_AREA    4
#define LB2_MESH_BAD_COUNT   8
typedef struct {
    double  surface_area;   /* S */
    int64_t last_count;     /* n_{n_tris - 1} (0 when S is bad) */
    int32_t status;         /* LB2_MESH_* bits */
    int32_t pad;
} lb2_mesh_info;
size_t lb2_mesh_sample_scratch_bytes(int64_t n_tris);
int lb2_mesh_sample_prepare(void* h, void* stream, const double* verts, int64_t n_verts, const int32_t* tris, int64_t n_tris,
                            int64_t n_points, double* area, lb2_mesh_info* d_info, void* scratch);
int lb2_mesh_sample_points(void* h, void* stream, const double* verts, const int32_t* tris, int64_t n_tris, const void* scratch,
                           const uint32_t* words, int64_t n_points, double* out);

/* ---- SemanticKITTI scene-completion (SSC) voxel grids (ssc.cu, lidiff_b200/ssc.py) — the format of the semantic-kitti-api
 * development kit (auxiliary/io_data.py, generate_sequential.py), restated; lidiff_b200/ssc.py holds the same constants.
 *
 * The grid is (256, 256, 32) voxels of 0.2 m in C order, v = (i 256 + j) 32 + k, over [min, max) with min = (0, -25.6, -2) and
 * max = (51.2, 25.6, 4.4), in the scan's frame.
 *   Packed bits (`.bin`, `.invalid`, 262 144 bytes): voxel v is bit 7 - (v & 7) of byte v >> 3 (MSB first).  On the device a grid
 *     is LB2_SSC_WORDS uint32 whose little-endian bytes are the file's bytes, so voxel v is bit (v & 31) ^ 7 of word v >> 5.
 *   Labels (`.label`): LB2_SSC_VOXELS little-endian uint16.  A voxel is occupied iff its label is neither 0 (empty) nor 255 (ignore).
 *   Voxel -> point: the centre, min_d + (idx_d + 0.5) 0.2 per axis in fp64 (the product and the sum each rounded).
 *   Point -> voxel: idx_d = floor((p_d - min_d) / 0.2) per axis in fp64 (difference and quotient each rounded); the point lies in the
 *     grid iff every idx_d is in [0, dim_d).  A row with a NaN / inf coordinate is dropped and counted, never clamped.
 *
 * lb2_ssc_grid_count: G grids (kind LB2_SSC_BITS: uint32[G][LB2_SSC_WORDS]; LB2_SSC_LABELS: uint16[G][LB2_SSC_VOXELS], device) ->
 *   offsets (device int64[G + 1]): offsets[0] = 0, offsets[g + 1] - offsets[g] = the occupied voxels of grid g; the per-word
 *   occupancy and in-grid positions stay in scratch (>= lb2_ssc_scratch_bytes(G), 16-byte aligned).  Three launches.
 * lb2_ssc_grid_points: out (device fp64 (offsets[G], 3)) = the centres of every grid's occupied voxels, grid after grid, each grid's
 *   in ascending v (np.nonzero's order), from the scratch of a grid_count call on the same G (one launch; no atomics: the same
 *   bytes on every run).  A caller reads offsets[G] in between to size out.
 * lb2_ssc_voxelize: G clouds, rows [offsets[g], offsets[g + 1]) of pts (device fp64 (n, 3); offsets device int64[G + 1],
 *   offsets[G] = n) -> bits (device uint32[G][LB2_SSC_WORDS], cleared first; each point's voxel set by atomicOr) and
 *   d_info[g] (device, cleared first): the rows dropped as non-finite and as outside the grid.
 * lb2_ssc_confusion: out (device int64[G][3]) = (TP, FP, FN) of predicted occupancy bits (uint32[G][LB2_SSC_WORDS]) against
 *   ground-truth labels (uint16[G][LB2_SSC_VOXELS]) over the valid voxels: a voxel is invalid when its label is 255 or its bit of
 *   `invalid` (uint32[G][LB2_SSC_WORDS], NULL: none) is set.  TP = pred & gt, FP = pred & !gt, FN = !pred & gt, gt = occupied.
 *   Integer popcounts; the same counts on every run. */
#define LB2_SSC_DIM_X   256
#define LB2_SSC_DIM_Y   256
#define LB2_SSC_DIM_Z   32
#define LB2_SSC_VOXELS  2097152      /* 256 x 256 x 32 */
#define LB2_SSC_WORDS   65536        /* LB2_SSC_VOXELS / 32 */
#define LB2_SSC_VOXEL   0.2
#define LB2_SSC_MIN_X   0.0
#define LB2_SSC_MIN_Y   (-25.6)
#define LB2_SSC_MIN_Z   (-2.0)
#define LB2_SSC_IGNORE  255
#define LB2_SSC_BITS    0
#define LB2_SSC_LABELS  1
typedef struct {
    int64_t non_finite;     /* rows with a NaN / inf coordinate */
    int64_t outside;        /* finite rows outside the grid */
} lb2_ssc_voxel_info;
size_t lb2_ssc_scratch_bytes(int64_t n_grids);
int lb2_ssc_grid_count(void* h, void* stream, const void* grids, int32_t kind, int64_t n_grids, int64_t* offsets, void* scratch);
int lb2_ssc_grid_points(void* h, void* stream, int64_t n_grids, const int64_t* offsets, const void* scratch, double* out);
int lb2_ssc_voxelize(void* h, void* stream, const double* pts, const int64_t* offsets, int64_t n_grids, int64_t n_points,
                     uint32_t* bits, lb2_ssc_voxel_info* d_info);
int lb2_ssc_confusion(void* h, void* stream, const uint32_t* pred_bits, const uint16_t* gt_labels, const uint32_t* invalid,
                      int64_t n_grids, int64_t* out);

#ifdef __cplusplus
}
#endif
#endif  /* LIDIFF_B200_H_ */
