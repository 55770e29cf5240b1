// K4 (variant C) — sparse convolution in gather-GEMM-scatter form on the tensor cores, for the levels
// where a voxel has only a few neighbours (L0-L2: 1.1 - 4.8 of 27).  The output-stationary variant
// (spconv_tc.cu) pays a full 128-row MMA for every (tile, offset) that has at least one pair; here the
// (in,out) pairs of a kernel offset are compacted first, so every MMA row is a real pair:
//
//   for each offset k (except the centre, which the output-stationary kernel handles as a dense GEMM):
//       Y[pairs_k, Cout] = X[pair_in] @ W[k]          wgmma, FP16x3 split, accumulator in registers
//       out[pair_out] += Y                             red.global.add.v2.f32
//
// Persistent, weight-stationary: one CTA per SM walks a contiguous range of 128-pair tiles (sorted by k), so
// the packed W[k] (all Cin chunks, <= 96 KB) is loaded into shared memory once per run of equal k and every
// MMA reads B from there; only the gathered A rows stream through the stage ring.
//   warpgroup 0   A producers (gather by pair_in, fp16 hi/lo split, SWIZZLE_128B image); thread 0 also loads W[k]
//                 (cp.async.bulk) at the start of every run of equal k
//   warpgroups 1, 2  consumers: pairs [0, 64) / [64, 128) of the tile, wgmma, then red.add of the rows to out[pair_out]
// The scattered buffer is the `pre_add` input of the centre convolution, which applies BN/ReLU/residual/gate.
// (A tile of one offset has at most 3 x 12 chained MMA steps: no two-level accumulation is needed.)
//
// Stands behind ME.MinkowskiConvolution forward (ME's own GPU algorithm is this gather-GEMM-scatter).
#include "common.cuh"
#include <algorithm>
#include "tc_common.cuh"

namespace sc {
using namespace tc;

constexpr int THREADS = 384;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int MAX_STAGES = 4;
constexpr int MAX_KVOL = 27;

struct Params {
    int c1, c2, cout, kvol, nchunks, stages, npass;
    const unsigned char* wpacked;
    const int* pair_in;
    const int* pair_out;
    const int* koff;        // [kvol+1]
    const int* tile_off;    // [kvol+1]
    const float* in1[2];
    const float* in2[2];
    const void* in1_h[2];
    const void* in2_h[2];
    float* out[2];
};

template <int N>
__global__ void __launch_bounds__(THREADS, 1) k_spconv_scatter(const Params p) {
    extern __shared__ unsigned char smem_raw[];
    __shared__ int s_koff[MAX_KVOL + 1];
    __shared__ int s_toff[MAX_KVOL + 1];
    __shared__ __align__(8) uint64_t bars[2 * MAX_STAGES + 2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ctot = p.c1 + p.c2;
    if (threadIdx.x <= p.kvol) { s_koff[threadIdx.x] = p.koff[threadIdx.x]; s_toff[threadIdx.x] = p.tile_off[threadIdx.x]; }

    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* gen = smem_raw + (base - raw);
    constexpr uint32_t b_tile = (uint32_t)N * 128u;
    const uint32_t w_bytes = (uint32_t)p.nchunks * 2u * b_tile;          // resident W[k]
    const uint32_t a_stage = 2u * A_TILE;
    unsigned char* a_gen = gen + w_bytes;
    const uint32_t a_base = base + w_bytes;
    const uint32_t bar0 = smem_u32(bars);
    auto full_a = [&](int s) { return bar0 + 8u * s; };
    auto empty_a = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };
    const uint32_t w_full = bar0 + 8u * (2 * MAX_STAGES), w_empty = bar0 + 8u * (2 * MAX_STAGES + 1);

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(full_a(s), 128); mbar_init(empty_a(s), NUM_CONSUMER_WARPS); }
        mbar_init(w_full, 1); mbar_init(w_empty, NUM_CONSUMER_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // this CTA's contiguous range of (pass, tile) work items
    const int tiles_per_pass = s_toff[p.kvol];
    const long long total = (long long)tiles_per_pass * p.npass;
    const int t_begin = (int)(total * blockIdx.x / gridDim.x), t_end = (int)(total * (blockIdx.x + 1) / gridDim.x);

    // decode work item T -> (pass, k, first pair, pair count)
    auto decode = [&](int T, int& pass, int& k, int& pbase, int& cnt) {
        pass = T / tiles_per_pass;
        const int t = T - pass * tiles_per_pass;
        k = 0;
        while (k + 1 < p.kvol && s_toff[k + 1] <= t) ++k;
        pbase = s_koff[k] + (t - s_toff[k]) * BM;
        cnt = min(BM, s_koff[k + 1] - pbase);
    };

    if (warp < 4) {
        // =========================== producers ===========================
        const int sub = threadIdx.x & 7, rbase = threadIdx.x >> 3;
        // cp.async lookahead: stages still landing while the next is issued.  S - 2, not S - 1: a consumer releases a stage only once it
        // holds the next one (wgmma_wait<1>), so the producers must be able to publish stage i + 1 while stage i - 1 is still held
        const int D = max(p.stages - 2, 0);
        int it = 0, arrived = 0, wrun = -1, cur_k = -1, cur_pass = -1;
        for (int T = t_begin; T < t_end; ++T) {
            int pass, k, pbase, cnt;
            decode(T, pass, k, pbase, cnt);
            if (threadIdx.x == 0 && (k != cur_k || pass != cur_pass)) {
                // new run of equal k: W[k] replaces the previous weights once the consumers are done with them.  The stages this
                // thread still owes an arrival are published first (the consumers finish the previous run only with them).
                cp_async_wait<0>();
                fence_proxy_async();
                for (; arrived < it; ++arrived) mbar_arrive(full_a(arrived % p.stages));
                ++wrun; cur_k = k; cur_pass = pass;
                if (wrun >= 1) mbar_wait(w_empty, (wrun - 1) & 1);
                const unsigned char* src = p.wpacked + PACK_HEADER + (size_t)k * w_bytes;
                mbar_expect_tx(w_full, w_bytes);
                for (int c = 0; c < p.nchunks; ++c) bulk_g2s(base + (uint32_t)c * 2u * b_tile, src + (size_t)c * 2u * b_tile, 2u * b_tile, w_full);
            }
            const bool use_h = (p.in1_h[pass] != nullptr) && (p.c2 == 0 || p.in2_h[pass] != nullptr);
            int src[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { const int r = rbase + 16 * j; src[j] = r < cnt ? __ldg(p.pair_in + pbase + r) : -1; }
            for (int c = 0; c < p.nchunks; ++c) {
                const int s = it % p.stages;
                mbar_wait(empty_a(s), ((it / p.stages) & 1) ^ 1);
                unsigned char* a_hi = a_gen + (size_t)s * a_stage;
                const uint32_t a_hi_u = a_base + (uint32_t)s * a_stage;
                const int ch = c * KC + sub * 8;
                if (ch < ctot) {
                    const bool first = ch < p.c1;
                    const int cw = first ? p.c1 : p.c2;
                    const int co = first ? ch : ch - p.c1;
                    if (use_h) produce_a_split(reinterpret_cast<const __half*>(first ? p.in1_h[pass] : p.in2_h[pass]), cw, co, src, a_hi_u, a_hi_u + A_TILE, rbase, sub);
                    else produce_a_f32(first ? p.in1[pass] : p.in2[pass], cw, co, src, a_hi, a_hi + A_TILE, rbase, sub);
                }
                // one protocol for both paths: a cp.async group per stage (empty for the fp32 path), published D stages later
                cp_async_commit();
                ++it;
                if (it - arrived > D) {
                    cp_async_wait_dyn(D);
                    fence_proxy_async();
                    mbar_arrive(full_a(arrived % p.stages));
                    ++arrived;
                }
            }
        }
        cp_async_wait<0>();
        fence_proxy_async();
        for (; arrived < it; ++arrived) mbar_arrive(full_a(arrived % p.stages));
    } else {
        // =========================== consumers: wgmma, then red.add into out[pair_out] ===========================
        const int wg = (warp >> 2) - 1;
        const float out_scale = __ldg(reinterpret_cast<const float*>(p.wpacked) + 1);
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // this thread's tile rows: r0 and r0 + 8
        float acc[N / 2];
        int it = 0, wrun = -1, cur_k = -1, cur_pass = -1;
        for (int T = t_begin; T < t_end; ++T) {
            int pass, k, pbase, cnt;
            decode(T, pass, k, pbase, cnt);
            if (k != cur_k || pass != cur_pass) {              // new run of equal k: its weights must have landed
                ++wrun; cur_k = k; cur_pass = pass;
                mbar_wait(w_full, wrun & 1);
            }
            const int orow0 = r0 < cnt ? __ldg(p.pair_out + pbase + r0) : -1;
            const int orow1 = r0 + 8 < cnt ? __ldg(p.pair_out + pbase + r0 + 8) : -1;
            int prev_s = -1;
            for (int c = 0; c < p.nchunks; ++c, ++it) {
                const int s = it % p.stages;
                mbar_wait(full_a(s), (it / p.stages) & 1);
                const uint32_t a_hi = a_base + (uint32_t)s * a_stage + (uint32_t)wg * (A_TILE / 2), a_lo = a_hi + A_TILE;
                const uint32_t b_hi = base + (uint32_t)c * 2u * b_tile, b_lo = b_hi + b_tile;
                const int ksteps = min(KC, ctot - c * KC) >> 4;
                reg_fence(acc);
                wg_stage_mma<N>(acc, a_hi, a_lo, b_hi, b_lo, ksteps, c == 0);
                reg_fence(acc);
                wgmma_wait<1>();
                if (prev_s >= 0 && lane == 0) mbar_arrive(empty_a(prev_s));
                prev_s = s;
            }
            wgmma_wait<0>();
            reg_fence(acc);
            if (lane == 0) mbar_arrive(empty_a(prev_s));
            // last tile of this run of equal k?  then the weights may be replaced
            bool run_ends = (T + 1 == t_end);
            if (!run_ends) {
                int p2, k2, pb2, c2;
                decode(T + 1, p2, k2, pb2, c2);
                run_ends = (k2 != k) || (p2 != pass);
            }
            if (run_ends && lane == 0) mbar_arrive(w_empty);
            float* out = p.out[pass];
#pragma unroll
            for (int i = 0; i < N / 2; i += 2) {
                const int orow = ((i >> 1) & 1) ? orow1 : orow0;
                if (orow < 0) continue;
                const int col = 8 * (i >> 2) + 2 * (lane & 3);
                asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(out + (long long)orow * p.cout + col),
                             "f"(acc[i] * out_scale), "f"(acc[i + 1] * out_scale) : "memory");
            }
        }
    }
}

// ---- pair lists of a kernel map, grouped by offset ------------------------------------------------------------------
__global__ void k_pair_count(const int* __restrict__ nbr, long long nbr_stride, const int* __restrict__ d_n, int n_cap, int skip_k,
                             int* __restrict__ cnt) {
    const int k = blockIdx.y;
    if (k == skip_k) return;
    const int n = d_n ? min(*d_n, n_cap) : n_cap;
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    const bool hit = o < n && nbr[(long long)k * nbr_stride + o] >= 0;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(cnt + k, __popc(m));
}

__global__ void k_pair_scan(const int* __restrict__ cnt, int kvol, int* __restrict__ koff, int* __restrict__ tile_off, int* __restrict__ cursor) {
    if (threadIdx.x == 0) {
        int a = 0, t = 0;
        for (int k = 0; k < kvol; ++k) { koff[k] = a; tile_off[k] = t; cursor[k] = 0; a += cnt[k]; t += (cnt[k] + tc::BM - 1) / tc::BM; }
        koff[kvol] = a; tile_off[kvol] = t;
    }
}

__global__ void k_pair_fill(const int* __restrict__ nbr, long long nbr_stride, const int* __restrict__ d_n, int n_cap, int skip_k,
                            const int* __restrict__ koff, int* __restrict__ cursor, int* __restrict__ pair_in, int* __restrict__ pair_out) {
    const int k = blockIdx.y;
    if (k == skip_k) return;
    const int n = d_n ? min(*d_n, n_cap) : n_cap;
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = o < n ? nbr[(long long)k * nbr_stride + o] : -1;
    const unsigned m = __ballot_sync(0xffffffffu, v >= 0);
    if (!m) return;
    const int lane = threadIdx.x & 31;
    int basep = 0;
    if (lane == __ffs(m) - 1) basep = atomicAdd(cursor + k, __popc(m));
    basep = __shfl_sync(0xffffffffu, basep, __ffs(m) - 1);
    if (v >= 0) {
        const int pos = koff[k] + basep + __popc(m & ((1u << lane) - 1));
        pair_in[pos] = v;
        pair_out[pos] = o;
    }
}

__global__ void k_zero_rows(float* __restrict__ buf, const int* __restrict__ d_n, int n_cap, int c) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int n = d_n ? min(*d_n, n_cap) : n_cap;
    if (t < (long long)n * c / 4) reinterpret_cast<float4*>(buf)[t] = make_float4(0.f, 0.f, 0.f, 0.f);
}

static size_t smem_bytes(int cin, int cout, int stages) {
    const int nchunks = (cin + tc::KC - 1) / tc::KC;
    return 1024 + (size_t)nchunks * 2 * cout * 128 + (size_t)stages * 2 * tc::A_TILE;
}

template <int N>
static int launch(Lb2Handle* h, cudaStream_t s, const Params& p, size_t smem) {
    cudaError_t e = lb2_configure_smem(h, LB2_K_SCATTER + (N / 32 - 1), k_spconv_scatter<N>, (int)(227 * 1024 - 512));   // static smem: bars + offsets
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "k_spconv_scatter smem attribute: %s", cudaGetErrorString(e));
    k_spconv_scatter<N><<<h->num_sms, THREADS, smem, s>>>(p);
    LB2_POST_LAUNCH(h, "k_spconv_scatter");
    return LB2_OK;
}

static bool shape_ok(int c1, int c2, int cout, int kvol) {
    const int ctot = c1 + c2;
    if (kvol < 1 || kvol > MAX_KVOL || ctot % 16 || ctot < 16) return false;
    if (c2 > 0 && (c1 % 8 || c2 % 8)) return false;
    if (cout % 32 || cout < 32 || cout > 128) return false;
    return smem_bytes(ctot, cout, 2) <= 227 * 1024 - 512;
}

}  // namespace sc

extern "C" size_t lb2_pair_list_scratch_bytes(void) { return 2 * 32 * sizeof(int); }

extern "C" int lb2_pair_list(void* handle, void* stream, const int32_t* nbr, int64_t nbr_stride, const int32_t* d_nout,
                             int32_t nout_cap, int32_t kvol, int32_t skip_k, int32_t* pair_in, int32_t* pair_out,
                             int32_t* koff, int32_t* tile_off, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && nbr && pair_in && pair_out && koff && tile_off && scratch && nout_cap > 0 && kvol >= 1 && kvol <= sc::MAX_KVOL, "pair_list");
    cudaStream_t s = (cudaStream_t)stream;
    int* cnt = (int*)scratch;
    int* cursor = cnt + 32;
    if (cudaMemsetAsync(cnt, 0, 64 * sizeof(int), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "pair_list memset%s", "");
    dim3 grid(cdiv(nout_cap, 256), kvol);
    sc::k_pair_count<<<grid, 256, 0, s>>>(nbr, nbr_stride, d_nout, nout_cap, skip_k, cnt);
    LB2_POST_LAUNCH(h, "k_pair_count");
    sc::k_pair_scan<<<1, 32, 0, s>>>(cnt, kvol, koff, tile_off, cursor);
    LB2_POST_LAUNCH(h, "k_pair_scan");
    sc::k_pair_fill<<<grid, 256, 0, s>>>(nbr, nbr_stride, d_nout, nout_cap, skip_k, koff, cursor, pair_in, pair_out);
    LB2_POST_LAUNCH(h, "k_pair_fill");
    return LB2_OK;
}

extern "C" int lb2_spconv_scatter_supported(int32_t c1, int32_t c2, int32_t cout, int32_t kvol) { return sc::shape_ok(c1, c2, cout, kvol) ? 1 : 0; }

extern "C" int lb2_spconv_scatter(void* handle, void* stream, const lb2_scatter_desc* d) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && d && d->weight_packed && d->pair_in && d->pair_out && d->koff && d->tile_off, "spconv_scatter null");
    LB2_REQUIRE(h, d->npass == 1 || d->npass == 2, "npass");
    if (!sc::shape_ok(d->c1, d->c2, d->cout, d->kvol)) return lb2_fail(h, LB2_ERR_UNSUP, "spconv_scatter: shape not supported%s", "");
    cudaStream_t s = (cudaStream_t)stream;
    sc::Params p;
    p.c1 = d->c1; p.c2 = d->c2; p.cout = d->cout; p.kvol = d->kvol; p.npass = d->npass;
    p.nchunks = (d->c1 + d->c2 + tc::KC - 1) / tc::KC;
    p.wpacked = (const unsigned char*)d->weight_packed;
    p.pair_in = d->pair_in; p.pair_out = d->pair_out; p.koff = d->koff; p.tile_off = d->tile_off;
    for (int i = 0; i < 2; ++i) {
        const int j = d->npass > 1 ? i : 0;
        LB2_REQUIRE(h, d->in1[j] && d->out[j] && ((d->c2 > 0) == (d->in2[j] != nullptr)), "spconv_scatter io");
        p.in1[i] = d->in1[j]; p.in2[i] = d->in2[j]; p.out[i] = d->out[j];
        p.in1_h[i] = d->in1_h[j]; p.in2_h[i] = d->in2_h[j];
    }
    int stages = sc::MAX_STAGES;
    while (stages > 2 && sc::smem_bytes(d->c1 + d->c2, d->cout, stages) > 227 * 1024 - 512) --stages;
    p.stages = stages;
    if (d->zero_rows_cap > 0) {        // clear the rows the scatter adds into
        for (int i = 0; i < d->npass; ++i) {
            sc::k_zero_rows<<<cdiv((long long)d->zero_rows_cap * d->cout / 4, 256), 256, 0, s>>>(d->out[i], d->d_zero_rows, d->zero_rows_cap, d->cout);
            LB2_POST_LAUNCH(h, "k_zero_rows");
        }
    }
    const size_t smem = sc::smem_bytes(d->c1 + d->c2, d->cout, stages);
    switch (d->cout) {
        case 32: return sc::launch<32>(h, s, p, smem);
        case 64: return sc::launch<64>(h, s, p, smem);
        case 96: return sc::launch<96>(h, s, p, smem);
        default: return sc::launch<128>(h, s, p, smem);
    }
}
