// K4 (variant B) — sparse convolution as an output-stationary implicit GEMM on the Hopper tensor
// cores (wgmma, accumulator in registers), split-precision FP16x3 so that 49 stacked layers stay
// inside the 1e-3 fp32 parity bar:
//     x = x_hi + x_lo (fp16 each),  w*2^k = w_hi + w_lo,   x.w ~= (x_hi.w_hi + x_lo.w_hi + x_hi.w_lo) * 2^-k
// (22 mantissa bits per operand; the dropped x_lo.w_lo term is ~2^-22 relative.  BF16x3 costs the same
// three MMAs and is far less accurate.  Weights are pre-scaled by a power of two per layer so their low
// parts stay in fp16's normal range.  Activations follow tc::split2: below |x| = 2^-3 the split has an
// absolute error floor of 2^-25; +-inf, NaN and any |x| >= 131024 make the products that read them non-finite.)
//
// A work item is 128 output rows x NC output channels of one guidance pass (NC = Cout, or Cout / 2 for Cout > 128).
// Items are numbered (tile slot, pass, channel half), the half fastest; slot i is tile tile_order[i] (most expensive
// first) when the map has a tile order.  The kernel is persistent: one CTA per SM, CTA b runs items b, b + G, b + 2G, ...
// (G = grid size) and stops at its first item past the live tiles.  The stage ring runs across items: the producers
// gather the next tile while the consumers finish the current one and run its epilogue.  Warp roles (384 threads):
//   warpgroup 0  producers: per item, first the tile's index table (one thread per row: output row, neighbour indices
//                of the offsets its row mask names, OR of the tile's offset mask) into one of two tile-info buffers;
//                then gather the neighbour rows of kernel offset k / channel chunk c (fp32 rows split to
//                fp16 hi/lo in registers, or the fp16 split companions with cp.async) into the K-major
//                SWIZZLE_128B shared-memory image; thread 0 also streams the pre-packed weight tiles of (k, c)
//                with cp.async.bulk (mbarrier complete_tx).  After a tile's last stage they publish one more ring
//                slot without loads, the epilogue slot, in which the consumers stage the tile's totals.
//                Runs on 88 registers per thread (setmaxnreg) so that the consumers can take 208.
//   warpgroups 1, 2  consumers: rows [0, 64) / [64, 128) of the tile, 3 x (chunk / 16) wgmma m64nNCk16 per stage.
//                TWO-LEVEL ACCUMULATION: a long chain of tensor-core accumulations loses accuracy linearly with
//                its length, so the chain is cut into groups of <= STEP_BUDGET MMA steps, each started from zero;
//                after each group the partial sum is added to a running fp32 total in registers (round-to-nearest).
//                The totals go through the epilogue slot to a coalesced epilogue:
//                BN affine + residual + ReLU + gate -> global.
// Kernel offsets where none of the tile's 128 rows has a neighbour are skipped by every role.
// OFFSET RANGES: a launch may run only the offsets [k0, k1) of a layer whose groups hold one offset each (range_mask = those bits).
// A row then starts its totals from partial_in when its mask has a bit below k0 (prior_mask), and a launch that is not the layer's
// last writes its unscaled totals to partial_out instead of running the epilogue.  The adds are those of one launch over all offsets,
// in the same order.
//
// Stands behind ME.MinkowskiConvolution(+Transpose) forward (lidiff/models/minkunet.py of the reference).
#include "common.cuh"
#include <algorithm>
#include <stdlib.h>
#include "tc_common.cuh"

namespace tc {

constexpr int THREADS = 384;
constexpr int NUM_PRODUCER = 128;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int STEP_BUDGET = 64;       // max chained MMA steps per accumulation group
constexpr int MAX_KVOL = 27;
constexpr int MAX_STAGES = 4;
constexpr int EPI_BATCH = 4;         // epilogue elements per lane whose loads are in flight together

struct Params {
    int c1, c2, cout, kvol;
    const unsigned char* wpacked;
    const float* scale;
    const float* shift;
    int relu;
    const int* nbr;
    long long nbr_stride;
    const int* d_mout;
    int mout_cap;
    const int* row_perm;
    const unsigned* row_mask;                           // per output row: bit k <=> nbr[k][row] >= 0; NULL = load every offset
    const int* tile_order;                              // tile of dispatch slot i, -1 = no live tile; NULL = natural order
    int stages, nchunks, group;                         // group: kernel offsets per accumulation group
    int npass, nsplit;
    lb2_conv_io io[2];
    uint32_t range_mask, prior_mask;                    // offsets of this launch / below it (~0u / 0 without a range)
    const float* partial_in;                            // (npass, mout_cap, cout) totals of the offsets below the range, or NULL
    float* partial_out;                                 // same layout: this launch's totals (no epilogue), or NULL
};

// Registers per thread after the producer warpgroup hands its surplus to the consumers.  The CTA is launched with 168 per thread
// (65536 / 384, rounded down to the allocation granule of 8); 128 * PRODUCER_REGS + 256 * CONSUMER_REGS must stay within 384 * 168.
// A consumer of NC = 128 holds 64 accumulator and 64 total registers; a producer of the fp32 path 16 float4 rows in flight.
constexpr int PRODUCER_REGS = 88;
constexpr int CONSUMER_REGS = 208;
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= THREADS * 168, "register split exceeds the CTA's allocation");

// What the producers know of a work item and the consumers need: written by the producers' prologue, read by the producers' gather
// (idx) and by the consumers (mask, item; row in the epilogue).  Two buffers, so that the next item's table is built while the
// consumers still run the current one.
struct TileInfo {
    int idx[MAX_KVOL * BM];      // neighbour row of (kernel offset k, tile row r) at [k * BM + r], -1 = none
    int row[BM];                 // output row of each tile row, -1 beyond the live rows
    uint32_t mask[4];            // per producer warp: OR of its rows' offset masks
    uint32_t prior[4];           // bit r & 31 of word r >> 5: tile row r starts from partial_in
    int item;                    // work item, -1 = this CTA has no more
    int pad[3];
};
// dynamic shared memory: 1024-byte alignment slack | stage ring | two tile-info buffers | mbarriers
constexpr int NUM_BARS = 3 * MAX_STAGES + 4;

template <int NC>
__global__ void __launch_bounds__(THREADS, 1) k_spconv_tc(const Params p) {
    extern __shared__ unsigned char smem_raw[];
    const int M = p.d_mout ? min(*p.d_mout, p.mout_cap) : p.mout_cap;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ctot = p.c1 + p.c2;
    const int S = p.stages;

    // ---- shared memory carve-up (tiles 1024-byte aligned for SWIZZLE_128B) -----------------------------
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* gen = smem_raw + (base - raw);
    constexpr uint32_t b_tile = (uint32_t)NC * 128u;                 // one fp16 B tile (hi or lo) of an item's channels
    const uint32_t b_full = (uint32_t)p.cout * 128u;                 // the same tile over all cout channels (packed layout)
    const uint32_t stage_bytes = 2u * A_TILE + 2u * b_tile;
    TileInfo* info = reinterpret_cast<TileInfo*>(gen + (size_t)S * stage_bytes);
    const uint32_t bar0 = smem_u32(info + 2);
    auto full_a = [&](int s) { return bar0 + 8u * s; };
    auto full_b = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };
    auto empty = [&](int s) { return bar0 + 8u * (2 * MAX_STAGES + s); };
    auto info_full = [&](int b) { return bar0 + 8u * (3 * MAX_STAGES + b); };
    auto info_empty = [&](int b) { return bar0 + 8u * (3 * MAX_STAGES + 2 + b); };

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(full_a(s), NUM_PRODUCER); mbar_init(full_b(s), 1); mbar_init(empty(s), NUM_CONSUMER_WARPS); }
        for (int b = 0; b < 2; ++b) { mbar_init(info_full(b), NUM_PRODUCER); mbar_init(info_empty(b), NUM_CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // Ring slot `it` (data stage or epilogue slot) is ring stage it % S in phase it / S; both roles count it across items.  Item j of
    // this CTA uses tile-info buffer j & 1 in phase j >> 1.
    if (warpgroup_role() == 0) {
        // =========================== producers: tile table, A gather (all 128 threads), B weights (thread 0) ===========================
        setmaxnreg_dec<PRODUCER_REGS>();
        const int sub = threadIdx.x & 7;           // 8-channel group inside the 64-channel chunk
        const int rbase = threadIdx.x >> 3;        // 0..15
        // cp.async lookahead: stages still landing while the next is issued.  S - 2, not S - 1: a consumer releases a stage only once it
        // holds the next one (wgmma_wait<1>), so the producers must be able to publish stage i + 1 while stage i - 1 is still held
        const int D = max(S - 2, 0);
        int it = 0, arrived = 0;
        // item x = (slot * npass + pass) * nsplit + half: the passes and channel halves of a tile are consecutive items and run on
        // neighbouring CTAs at the same time (their gathers of the same neighbour rows meet in L2); slots follow the tile order, most
        // expensive tile first, when there is one, so the static stride deals the tiles roughly longest first
        auto tile_of = [&](int x) {
            const int slot_i = x / (p.nsplit * p.npass);
            return slot_i * BM >= p.mout_cap ? -1 : p.tile_order ? __ldg(p.tile_order + slot_i) : slot_i;
        };
        // index loads of tile row threadIdx.x: its output row and the neighbour row of every kernel offset (-1 = none).  The row's
        // neighbour mask names the offsets that have an entry: only those index loads are issued, all at once (the sparse levels' rows
        // have a few of 27, and the loads hit random rows of the map).  Without a mask every offset is loaded.  A row whose mask has an
        // offset below the launch's range (it starts from partial_in) gets bit 30 of `row` set (rows < 2^22), so that no register
        // lives across the loop for it.
        auto load_row = [&](int tile) {
            const int slot = tile * BM + threadIdx.x;
            return (tile >= 0 && slot < M) ? (p.row_perm ? __ldg(p.row_perm + slot) : slot) : -1;
        };
        auto load_indices = [&](int& row, int (&v)[MAX_KVOL]) {
            const uint32_t m = row < 0 ? 0u : (p.row_mask ? __ldg(p.row_mask + row) : ~0u);
            const uint32_t want = m & p.range_mask;
#pragma unroll
            for (int k = 0; k < MAX_KVOL; ++k) {
                v[k] = -1;
                if (k < p.kvol && (want >> k) & 1u) v[k] = p.nbr ? __ldg(p.nbr + (long long)k * p.nbr_stride + row) : row;
            }
            if (m & p.prior_mask) row |= 1 << 30;         // after the index loads, which address with the plain row
        };
        int x = blockIdx.x, tile = tile_of(x), row = load_row(tile), v[MAX_KVOL];
        load_indices(row, v);
        for (int j = 0;; ++j) {
            TileInfo& ti = info[j & 1];
            mbar_wait(info_empty(j & 1), ((j >> 1) & 1) ^ 1);
            if (tile < 0 || tile * BM >= M) {      // the dead items are the last ones: this CTA is done
                if (threadIdx.x == 0) ti.item = -1;
                mbar_arrive(info_full(j & 1));
                break;
            }
            // ---- the tile's index table + mask of non-empty kernel offsets: one thread per tile row ----
            {
                ti.row[threadIdx.x] = row < 0 ? row : row & ~(1 << 30);
                uint32_t have = 0;
#pragma unroll
                for (int k = 0; k < MAX_KVOL; ++k) {
                    if (k < p.kvol) {
                        ti.idx[k * BM + threadIdx.x] = v[k];
                        if (v[k] >= 0) have |= 1u << k;
                    }
                }
                const uint32_t wmask = __reduce_or_sync(0xffffffffu, have);
                const uint32_t wprior = __ballot_sync(0xffffffffu, row >= 0 && (row >> 30));
                if (lane == 0) { ti.mask[warp] = wmask; ti.prior[warp] = wprior; }
                if (threadIdx.x == 0) ti.item = x;
            }
            mbar_arrive(info_full(j & 1));
            mbar_wait(info_full(j & 1), (j >> 1) & 1);         // the other producer warps' rows and masks
            const uint32_t kmask = ti.mask[0] | ti.mask[1] | ti.mask[2] | ti.mask[3];
            const int x_next = x + gridDim.x;
            const int tile_next = tile_of(x_next);              // loaded now, used after the tile's stages
            const int n0 = (x % p.nsplit) * NC;                 // first output channel of the item
            const lb2_conv_io io = p.io[(x / p.nsplit) % p.npass];
            const bool use_h = (io.in1_h != nullptr) && (p.c2 == 0 || io.in2_h != nullptr);   // fp16 split inputs: cp.async gather
            for (uint32_t km = kmask; km; km &= km - 1) {
                const int k = __ffs(km) - 1;
                const int* idxk = ti.idx + k * BM;
                int src[8];
#pragma unroll
                for (int r = 0; r < 8; ++r) src[r] = idxk[rbase + 16 * r];
                for (int c = 0; c < p.nchunks; ++c) {
                    const int s = it % S;
                    mbar_wait(empty(s), ((it / S) & 1) ^ 1);
                    unsigned char* a_hi = gen + (size_t)s * stage_bytes;
                    const uint32_t a_hi_u = base + (uint32_t)s * stage_bytes;
                    if (threadIdx.x == 0) {
                        const uint32_t dst = a_hi_u + 2u * A_TILE;
                        const unsigned char* wsrc = p.wpacked + PACK_HEADER + ((size_t)k * p.nchunks + c) * (2u * b_full) + (size_t)n0 * 128u;
                        mbar_expect_tx(full_b(s), 2u * b_tile);
                        bulk_g2s(dst, wsrc, b_tile, full_b(s));                      // hi rows n0 .. n0+NC
                        bulk_g2s(dst + b_tile, wsrc + b_full, b_tile, full_b(s));    // lo rows
                    }
                    const int ch = c * KC + sub * 8;
                    if (ch < ctot) {
                        const bool first = ch < p.c1;
                        const int cw = first ? p.c1 : p.c2;
                        const int co = first ? ch : ch - p.c1;
                        if (use_h) produce_a_split(reinterpret_cast<const __half*>(first ? io.in1_h : io.in2_h), cw, co, src, a_hi_u, a_hi_u + A_TILE, rbase, sub);
                        else produce_a_f32(first ? io.in1 : io.in2, cw, co, src, a_hi, a_hi + A_TILE, rbase, sub);
                    }
                    // one protocol for both paths (consecutive items may take different ones): a cp.async group per stage (empty for the
                    // fp32 path), published D stages later
                    cp_async_commit();
                    ++it;
                    if (it - arrived > D) {
                        cp_async_wait_dyn(D);
                        fence_proxy_async();
                        mbar_arrive(full_a(arrived % S));
                        ++arrived;
                    }
                }
            }
            // the epilogue slot: no loads, the consumers stage the tile's totals in it.  Then everything still owed is published, so
            // neither the tile's last stages nor its epilogue wait for the next tile's index loads.
            const int s = it % S;
            mbar_wait(empty(s), ((it / S) & 1) ^ 1);
            if (threadIdx.x == 0) mbar_arrive(full_b(s));
            ++it;
            x = x_next;
            tile = tile_next;
            row = load_row(tile);                  // in flight while the last stages land
            cp_async_wait<0>();
            fence_proxy_async();
            for (; arrived < it; ++arrived) mbar_arrive(full_a(arrived % S));
            load_indices(row, v);
        }
    } else {
        // =========================== consumers: wgmma + two-level accumulation, epilogue ===========================
        setmaxnreg_inc<CONSUMER_REGS>();
        const int wg = (warp >> 2) - 1;                           // 0: tile rows [0, 64), 1: rows [64, 128)
        const float out_scale = __ldg(reinterpret_cast<const float*>(p.wpacked) + 1);     // 2^-k of the packed weights
        int it = 0;
        for (int j = 0;; ++j) {
            const TileInfo& ti = info[j & 1];
            mbar_wait(info_full(j & 1), (j >> 1) & 1);
            const int x = ti.item;
            if (x < 0) break;
            const int n_off = __popc(ti.mask[0] | ti.mask[1] | ti.mask[2] | ti.mask[3]);
            // tot starts at -0: -0 + x == x for every x (+0 and -0 included), so the first fold is an exact copy without a select.
            // A row of a range launch with offsets below the range starts from the totals they left in partial_in.
            float acc[NC / 2], tot[NC / 2];
            if (p.partial_in) {
                const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // this thread's fragment rows: r0, r0 + 8
                const float* src[2];
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int rr = r0 + 8 * hh;
                    const bool pr = (ti.prior[rr >> 5] >> (rr & 31)) & 1u;
                    src[hh] = pr ? p.partial_in + ((long long)((x / p.nsplit) % p.npass) * p.mout_cap + ti.row[rr]) * p.cout + (x % p.nsplit) * NC
                                 : nullptr;
                }
#pragma unroll
                for (int i = 0; i < NC / 2; i += 2) {
                    const float* q = src[(i >> 1) & 1];
                    const float2 t = q ? __ldcg(reinterpret_cast<const float2*>(q + 8 * (i >> 2) + 2 * (lane & 3))) : make_float2(-0.f, -0.f);
                    tot[i] = t.x;
                    tot[i + 1] = t.y;
                }
            } else {
#pragma unroll
                for (int i = 0; i < NC / 2; ++i) tot[i] = -0.f;
            }
            // one flat loop over the tile's stages (offset-major, chunk-minor), the stage sequence the producers publish
            const int n_it = n_off * p.nchunks;
            int c = 0, in_group = 0, off_idx = 0, prev_s = -1;
            for (int i = 0; i < n_it; ++i, ++it) {
                const int s = it % S;
                const uint32_t par = (it / S) & 1;
                mbar_wait(full_b(s), par);
                mbar_wait(full_a(s), par);
                const uint32_t a_hi = base + (uint32_t)s * stage_bytes + (uint32_t)wg * (A_TILE / 2), a_lo = a_hi + A_TILE;
                const uint32_t b_hi = base + (uint32_t)s * stage_bytes + 2u * A_TILE, b_lo = b_hi + b_tile;
                const int ksteps = min(KC, ctot - c * KC) >> 4;
                reg_fence(acc);
                wg_stage_mma<NC>(acc, a_hi, a_lo, b_hi, b_lo, ksteps, in_group == 0 && c == 0);   // first MMA of a group overwrites
                reg_fence(acc);
                wgmma_wait<1>();                                      // the MMAs of the previous stage are done: release it
                if (prev_s >= 0 && lane == 0) mbar_arrive(empty(prev_s));
                prev_s = s;
                if (++c < p.nchunks) continue;
                c = 0;
                ++off_idx;
                if (++in_group == p.group || off_idx == n_off) {      // partial sum of this group complete -> running total
                    wgmma_wait<0>();
                    reg_fence(acc);
                    if (lane == 0) mbar_arrive(empty(prev_s));
                    prev_s = -1;
#pragma unroll
                    for (int i = 0; i < NC / 2; ++i) tot[i] = __fadd_rn(tot[i], acc[i]);
                    in_group = 0;
                }
            }
            // the last stage always ends a group, so nothing is in flight here; ptxas cannot see that, and without this wait it injects one
            // on the loop's exit edge (C7517) before the epilogue reuses the accumulator registers
            wgmma_wait<0>();
            // ---- totals -> the epilogue slot, [BM][NC] fp32 with the 16-byte column chunks XOR-swizzled by row (no bank conflicts on
            //      the fragment writes nor the row reads; NC = 128 fills a stage exactly) ----------
            const int se = it % S;
            mbar_wait(full_b(se), (it / S) & 1);
            mbar_wait(full_a(se), (it / S) & 1);
            ++it;
            float* stage_c = reinterpret_cast<float*>(gen + (size_t)se * stage_bytes);
            {
                const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
                const float sc = p.partial_out ? 1.f : out_scale;         // partial totals stay unscaled (x * 1 == x)
#pragma unroll
                for (int i = 0; i < NC / 2; i += 2) {
                    const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3);
                    *reinterpret_cast<float2*>(stage_c + row * NC + (((col >> 2) ^ (row & 7)) << 2) + (col & 3)) =
                        make_float2(tot[i] * sc, tot[i + 1] * sc);
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // ---- epilogue, coalesced: consumer warp cw owns tile rows cw, cw + 8, ... and walks their (row, 4-channel) elements with
            //      consecutive lanes on consecutive channels, so every global access is a contiguous row segment.  A lane takes its
            //      elements in batches of EPI_BATCH: every load of a batch (pre_add, BN affine, residual, gate index) is issued before
            //      any of its arithmetic, the gate rows right after their indices, then the stores.  One element at a time, each
            //      element waited for its loads and its gate index -> gate row chain in turn, with the tensor cores idle.  The
            //      arithmetic of an element is unchanged.  ----------
            const lb2_conv_io io = p.io[(x / p.nsplit) % p.npass];
            const int n0 = (x % p.nsplit) * NC;                        // first output channel of the item
            const int cw = warp - 4;
            constexpr int nv = NC >> 2;                                // float4 per row (the item's channels)
            constexpr int PER_LANE = (BM / NUM_CONSUMER_WARPS) * nv / 32;
            static_assert(PER_LANE % EPI_BATCH == 0, "a lane's elements come in whole batches");
            const bool has_res = io.residual || io.residual_h;
            const bool gated = io.out_gated || io.out_gated_h;
            const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.partial_out) {        // a range launch that is not the layer's last: the totals only, coalesced as below
                float* dst = p.partial_out + (long long)((x / p.nsplit) % p.npass) * p.mout_cap * p.cout;
                for (int e = lane; e < PER_LANE * 32; e += 32) {
                    const int rr = cw + NUM_CONSUMER_WARPS * (e / nv);
                    const int lcol = (e % nv) * 4;
                    const int orow = ti.row[rr];
                    if (orow >= 0)
                        __stcg(reinterpret_cast<float4*>(dst + (long long)orow * p.cout + n0 + lcol),
                               *reinterpret_cast<const float4*>(stage_c + rr * NC + (((lcol >> 2) ^ (rr & 7)) << 2)));
                }
            }
            for (int e0 = 0; !p.partial_out && e0 < PER_LANE; e0 += EPI_BATCH) {
                int orow[EPI_BATCH], col[EPI_BATCH];
                long long gi[EPI_BATCH];
                float4 a4[EPI_BATCH], pre4[EPI_BATCH], s4[EPI_BATCH], h4[EPI_BATCH], res4[EPI_BATCH], g4[EPI_BATCH];
#pragma unroll
                for (int b = 0; b < EPI_BATCH; ++b) {
                    const int e = lane + 32 * (e0 + b);
                    const int rr = cw + NUM_CONSUMER_WARPS * (e / nv);
                    const int lcol = (e % nv) * 4;
                    col[b] = n0 + lcol;
                    orow[b] = ti.row[rr];
                    const bool live = orow[b] >= 0;
                    const long long ro = (long long)orow[b] * p.cout;
                    a4[b] = *reinterpret_cast<const float4*>(stage_c + rr * NC + (((lcol >> 2) ^ (rr & 7)) << 2));
                    pre4[b] = (live && io.pre_add) ? __ldg(reinterpret_cast<const float4*>(io.pre_add + ro + col[b])) : zero4;
                    s4[b] = p.scale ? __ldg(reinterpret_cast<const float4*>(p.scale + col[b])) : zero4;
                    h4[b] = p.scale ? __ldg(reinterpret_cast<const float4*>(p.shift + col[b])) : zero4;
                    res4[b] = (live && has_res) ? load_residual4(io.residual, io.residual_h, orow[b], p.cout, col[b]) : zero4;
                    gi[b] = (live && gated && io.gate_table && io.gate_idx) ? __ldg(io.gate_idx + orow[b]) : 0;
                }
#pragma unroll
                for (int b = 0; b < EPI_BATCH; ++b)
                    g4[b] = (orow[b] >= 0 && gated && io.gate_table) ? __ldg(reinterpret_cast<const float4*>(io.gate_table + gi[b] * p.cout + col[b])) : zero4;
#pragma unroll
                for (int b = 0; b < EPI_BATCH; ++b) {
                    if (orow[b] < 0) continue;
                    const long long ro = (long long)orow[b] * p.cout;
                    float y[4] = {a4[b].x, a4[b].y, a4[b].z, a4[b].w};
                    if (io.pre_add) {
                        y[0] += pre4[b].x; y[1] += pre4[b].y; y[2] += pre4[b].z; y[3] += pre4[b].w;
                    }
                    if (p.scale) {
                        y[0] = fmaf(y[0], s4[b].x, h4[b].x); y[1] = fmaf(y[1], s4[b].y, h4[b].y);
                        y[2] = fmaf(y[2], s4[b].z, h4[b].z); y[3] = fmaf(y[3], s4[b].w, h4[b].w);
                    }
                    if (has_res) {
                        y[0] += res4[b].x; y[1] += res4[b].y; y[2] += res4[b].z; y[3] += res4[b].w;
                    }
                    if (p.relu) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) y[q] = fmaxf(y[q], 0.f);
                    }
                    if (io.out) *reinterpret_cast<float4*>(io.out + ro + col[b]) = make_float4(y[0], y[1], y[2], y[3]);
                    if (io.out_h) store_split4(io.out_h, orow[b], p.cout, col[b], y);
                    if (gated) {
                        if (io.gate_table) {
                            y[0] *= g4[b].x; y[1] *= g4[b].y; y[2] *= g4[b].z; y[3] *= g4[b].w;
                        }
                        if (io.out_gated) *reinterpret_cast<float4*>(io.out_gated + ro + col[b]) = make_float4(y[0], y[1], y[2], y[3]);
                        if (io.out_gated_h) store_split4(io.out_gated_h, orow[b], p.cout, col[b], y);
                    }
                }
            }
            // the slot's next bulk copy is an async-proxy write after these generic accesses
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(empty(se));
                mbar_arrive(info_empty(j & 1));
            }
        }
    }
}

// ---- weight packing: (kvol, cin, cout) fp32 -> [256 B header][per (k, chunk): hi tile | lo tile], each tile cout rows
// x 128 B in the K-major SWIZZLE_128B image, channels beyond cin zero-filled.  Values are W * 2^k with k chosen so
// that max|W| * 2^k lies in [8192, 16384) (k_weight_absmax, weight_scale); header[1] = 2^-k is applied to the accumulator in the
// epilogue. ---------
__global__ void k_pack_weights(const float* __restrict__ w, int kvol, int cin, int cout, int nchunks, unsigned char* __restrict__ out) {
    const long long total = (long long)kvol * nchunks * cout * KC;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const float scale = weight_scale(*reinterpret_cast<const unsigned*>(out));
    if (t == 0) reinterpret_cast<float*>(out)[1] = 1.0f / scale;
    if (t >= total) return;
    const int kk = (int)(t % KC);
    const int n = (int)((t / KC) % cout);
    const int c = (int)((t / ((long long)KC * cout)) % nchunks);
    const int k = (int)(t / ((long long)KC * cout * nchunks));
    const int ch = c * KC + kk;
    const float v = ch < cin ? w[((long long)k * cin + ch) * cout + n] * scale : 0.f;
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(hi));
    const size_t tile = (size_t)cout * 128;
    unsigned char* blob = out + PACK_HEADER + ((size_t)k * nchunks + c) * 2 * tile;
    const uint32_t off = sw128(n, kk >> 3) + (uint32_t)(kk & 7) * 2u;
    *reinterpret_cast<__half*>(blob + off) = hi;
    *reinterpret_cast<__half*>(blob + tile + off) = lo;
}

static bool shape_ok(int c1, int c2, int cout, int kvol) {
    const int ctot = c1 + c2;
    if (kvol < 1 || kvol > MAX_KVOL) return false;
    if (ctot % 16 != 0 || ctot < 16) return false;
    if (c2 > 0 && (c1 % 8 != 0 || c2 % 8 != 0)) return false;
    if (cout % 32 != 0 || cout < 32 || cout > 256) return false;
    if (cout > 128 && cout != 256) return false;        // Cout > 128 runs as two CTAs of Cout / 2: 256 only (128 per CTA)
    return true;
}

static size_t smem_bytes(int nc, int stages) {
    return 1024 + (size_t)stages * (2 * A_TILE + 2 * (size_t)nc * 128) + 2 * sizeof(TileInfo) + NUM_BARS * sizeof(uint64_t);
}

template <int NC>
static int launch(Lb2Handle* h, cudaStream_t s, const Params& p, int stages) {
    const size_t smem = smem_bytes(NC, stages);
    cudaError_t e = lb2_configure_smem(h, LB2_K_TC + (NC / 32 - 1), k_spconv_tc<NC>, (int)(227 * 1024));
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "k_spconv_tc smem attribute: %s", cudaGetErrorString(e));
    // persistent: one CTA per SM, or one per work item when there are fewer
    const unsigned grid = (unsigned)std::min<long long>(h->num_sms, (long long)cdiv(p.mout_cap, BM) * p.npass * p.nsplit);
    k_spconv_tc<NC><<<grid, THREADS, smem, s>>>(p);
    LB2_POST_LAUNCH(h, "k_spconv_tc");
    return LB2_OK;
}

}  // namespace tc

bool lb2_spconv_tc_supported(const lb2_conv_desc* d) { return tc::shape_ok(d->c1, d->c2, d->cout, d->kvol); }

extern "C" size_t lb2_packed_weight_bytes(int32_t kvol, int32_t cin, int32_t cout) {
    if (!tc::shape_ok(cin, 0, cout, kvol)) return 0;
    const int nchunks = (cin + tc::KC - 1) / tc::KC;
    return tc::PACK_HEADER + (size_t)kvol * nchunks * 2 * (size_t)cout * 128;
}

extern "C" int lb2_pack_weights(void* handle, void* stream, const float* weight, int32_t kvol, int32_t cin, int32_t cout, void* packed) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && weight && packed, "pack_weights null");
    if (!tc::shape_ok(cin, 0, cout, kvol)) return lb2_fail(h, LB2_ERR_UNSUP, "pack_weights: shape not supported by the tensor-core variant%s", "");
    const int nchunks = (cin + tc::KC - 1) / tc::KC;
    const long long total = (long long)kvol * nchunks * cout * tc::KC;
    const long long nw = (long long)kvol * cin * cout;
    if (cudaMemsetAsync(packed, 0, tc::PACK_HEADER, (cudaStream_t)stream) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "pack_weights memset%s", "");
    tc::k_weight_absmax<<<(unsigned)std::min<long long>(cdiv(nw, 256), 1024), 256, 0, (cudaStream_t)stream>>>(weight, nw, (unsigned*)packed);
    LB2_POST_LAUNCH(h, "k_weight_absmax");
    tc::k_pack_weights<<<cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(weight, kvol, cin, cout, nchunks, (unsigned char*)packed);
    LB2_POST_LAUNCH(h, "k_pack_weights");
    return LB2_OK;
}

int lb2_spconv_tc_launch(Lb2Handle* h, cudaStream_t s, const lb2_conv_desc* d) {
    tc::Params p;
    p.c1 = d->c1; p.c2 = d->c2; p.cout = d->cout; p.kvol = d->kvol;
    p.wpacked = (const unsigned char*)d->weight_packed;
    p.scale = d->scale; p.shift = d->shift; p.relu = d->relu;
    p.nbr = d->nbr; p.nbr_stride = d->nbr_stride; p.d_mout = d->d_mout; p.mout_cap = d->mout_cap; p.row_perm = d->row_perm;
    p.tile_order = d->nbr ? d->tile_order128 : nullptr;     // the tile order ranks the tiles of a map's row order
    p.row_mask = d->nbr ? (const unsigned*)d->row_mask : nullptr;
    p.nchunks = (d->c1 + d->c2 + tc::KC - 1) / tc::KC;
    // a consumer thread holds NC / 2 accumulator and NC / 2 total registers: NC <= 128, so Cout 256 runs as two CTAs of 128 channels
    const int nsplit = d->cout > 128 ? 2 : 1;
    const int nc = d->cout / nsplit;
    p.npass = d->npass > 1 ? 2 : 1;
    p.nsplit = nsplit;
    int stages = tc::MAX_STAGES;
    while (stages > 2 && tc::smem_bytes(nc, stages) > 227 * 1024) --stages;
    p.stages = stages;
    const int steps_per_offset = 3 * ((d->c1 + d->c2 + 15) / 16);
    p.group = std::max(1, tc::STEP_BUDGET / steps_per_offset);
    p.io[0] = d->io[0]; p.io[1] = d->io[d->npass > 1 ? 1 : 0];
    p.range_mask = ~0u; p.prior_mask = 0u; p.partial_in = nullptr; p.partial_out = nullptr;
    if (d->k1 > 0) {
        // the same bits as one launch need one offset per accumulation group: then every offset is one RN add to the total
        if (d->kvol != 27 || !d->nbr || !d->row_mask || d->k0 < 0 || d->k0 >= d->k1 || d->k1 > 27 || p.group != 1 ||
            (d->k0 > 0) != (d->partial_in != nullptr) || (d->k1 < 27) != (d->partial_out != nullptr))
            return lb2_fail(h, LB2_ERR_ARG, "offset range: needs kvol 27, a map with row masks, c1 + c2 >= 176, 0 <= k0 < k1 <= 27, "
                                            "partial_in iff k0 > 0 and partial_out iff k1 < 27%s", "");
        p.range_mask = ((1u << d->k1) - 1u) & ~((1u << d->k0) - 1u);
        p.prior_mask = (1u << d->k0) - 1u;
        p.partial_in = d->partial_in;
        p.partial_out = d->partial_out;
    }
    switch (nc) {
        case 32: return tc::launch<32>(h, s, p, stages);
        case 64: return tc::launch<64>(h, s, p, stages);
        case 96: return tc::launch<96>(h, s, p, stages);
        case 128: return tc::launch<128>(h, s, p, stages);
        default: return lb2_fail(h, LB2_ERR_UNSUP, "tensor-core variant: no kernel for %s output channels per CTA", nc == 80 ? "80" : nc == 112 ? "112" : "this many");
    }
}
