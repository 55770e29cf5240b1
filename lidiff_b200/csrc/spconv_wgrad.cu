// Weight gradient of the sparse convolution on the Hopper tensor cores (wgmma, accumulators in registers):
//     dW[k] (cin x cout) = sum_o X[nbr[k][o]]^T G[o]          (absent neighbours contribute nothing; nbr == NULL: identity, kvol 1)
// a gather-GEMM whose reduction dimension is the output rows.  The FP16x3 split is the forward's (spconv_tc.cu): X is split like an
// activation (tc::split2), G like a weight, after a power-of-two pre-scale that puts max|G| * 2^k in [8192, 16384) (k_weight_absmax,
// weight_scale); the products are x_hi.g_hi + x_lo.g_hi + x_hi.g_lo.
//
// A CTA owns one (row chunk, offset k, 128 input channels, NC = 32 or 64 output channels) block.  Row chunks are a fixed function of the row
// count, each CTA writes its own fp32 partial dW, and k_wgrad_reduce adds the partials in chunk order: no float atomics, the same bits
// on every run.  Warp roles (384 threads):
//   warpgroup 0  producers: per stage 64 output rows; lane l takes rows 2l, 2l + 1 and, per 8-channel group, loads the fp32 rows of X
//                (neighbours) and G, splits them to fp16 hi/lo in registers and stores each channel's pair of rows as one 32-bit word,
//                so that the shared-memory images are K-major (K = rows) SWIZZLE_128B tiles: A = 128 channels of X^T, B = NC
//                channels of G^T.  A stage where no row has a neighbour is published empty and issues no MMAs.
//   warpgroups 1, 2  consumers: input channels [0, 64) / [64, 128) of the block, 3 x 4 wgmma m64nNCk16 per stage, partial sums cut
//                into groups of GROUP stages (the forward's two-level accumulation), folded into fp32 totals.
#include "common.cuh"
#include <algorithm>
#include "tc_common.cuh"

namespace tc {
namespace wgrad {

constexpr int THREADS = 384;
constexpr int NUM_PRODUCER = 128;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int BR = 64;                  // output rows (the GEMM's K) per stage: one 128-byte swizzle row of fp16
constexpr int GROUP = 5;                // stages per accumulation group: 5 x 12 MMA steps, within the forward's budget of 64
constexpr int MAX_STAGES = 4;
constexpr int MAX_CHUNKS = 16;
constexpr int CHUNK_ROWS = 8192;        // rows per chunk before the chunk count saturates
constexpr int PRODUCER_REGS = 88;
constexpr int CONSUMER_REGS = 208;
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= THREADS * 168, "register split exceeds the CTA's allocation");

struct Params {
    const float* x;            // (rows_in, cin)
    const float* g;            // (m_out, cout)
    const int* nbr;            // [kvol][nbr_stride] or NULL
    long long nbr_stride;
    int cin, cout, kvol, m_out;
    int rows_per_chunk, mblocks, nsplit, stages;
    const unsigned* header;    // [0] max|G| bits
    float* partial;            // (nchunks, kvol, cin, cout)
};

static int nchunks_of(int m_out) { return std::max(1, std::min(MAX_CHUNKS, (int)cdiv(m_out, CHUNK_ROWS))); }
static int rows_per_chunk_of(int m_out) { return (int)cdiv(cdiv(std::max(m_out, 1), nchunks_of(m_out)), BR) * BR; }

// 8 consecutive channels [ch, ch + 8) of row `src` of a (rows, c) fp32 matrix, times `mul`; zeros for src < 0 and past c
__device__ __forceinline__ void load8(const float* __restrict__ base, int c, int src, int ch, float mul, float (&v)[8]) {
    if (src >= 0 && ch + 8 <= c && (c & 3) == 0) {
        const float4* rp = reinterpret_cast<const float4*>(base + (long long)src * c + ch);
        const float4 a = __ldg(rp), b = __ldg(rp + 1);
        v[0] = a.x * mul; v[1] = a.y * mul; v[2] = a.z * mul; v[3] = a.w * mul;
        v[4] = b.x * mul; v[5] = b.y * mul; v[6] = b.z * mul; v[7] = b.w * mul;
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (src >= 0 && ch + j < c) ? __ldg(base + (long long)src * c + ch + j) * mul : 0.f;
    }
}

// channels [row0, row0 + 8) of the K-major images at K positions 2 pr, 2 pr + 1 (rows r0 -> v0, r1 -> v1): one 32-bit word each
__device__ __forceinline__ void store_pairs8(unsigned char* hi, unsigned char* lo, int row0, int pr, const float (&v0)[8], const float (&v1)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        uint32_t h, l;
        split2(v0[j], v1[j], h, l);
        const uint32_t off = sw128(row0 + j, pr >> 2) + (uint32_t)(pr & 3) * 4u;
        *reinterpret_cast<uint32_t*>(hi + off) = h;
        *reinterpret_cast<uint32_t*>(lo + off) = l;
    }
}

template <int NC>
__global__ void __launch_bounds__(THREADS, 1) k_spconv_wgrad(const Params p) {
    extern __shared__ unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int b = blockIdx.x;
    const int ns = b % p.nsplit; b /= p.nsplit;
    const int mb = b % p.mblocks; b /= p.mblocks;
    const int k = b % p.kvol;
    const int chunk = b / p.kvol;
    const int m0 = mb * BM, n0 = ns * NC;
    const int r_begin = chunk * p.rows_per_chunk;
    const int r_end = min(p.m_out, r_begin + p.rows_per_chunk);
    const int nst = r_end > r_begin ? (r_end - r_begin + BR - 1) / BR : 0;
    const int S = p.stages;

    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* gen = smem_raw + (base - raw);
    constexpr uint32_t b_tile = (uint32_t)NC * 128u;
    constexpr uint32_t stage_bytes = 2u * A_TILE + 2u * b_tile;
    int* live = reinterpret_cast<int*>(gen + (size_t)S * stage_bytes);       // per stage: some row of it has a neighbour
    const uint32_t bar0 = smem_u32(live + MAX_STAGES);
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto empty = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(full(s), NUM_PRODUCER); mbar_init(empty(s), NUM_CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warpgroup_role() == 0) {
        // =========================== producers ===========================
        setmaxnreg_dec<PRODUCER_REGS>();
        const float gs = weight_scale(__ldg(p.header));
        const int pr = lane;
        for (int i = 0; i < nst; ++i) {
            const int s = i % S;
            mbar_wait(empty(s), ((i / S) & 1) ^ 1);
            const int o0 = r_begin + i * BR + 2 * pr;
            int src[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int o = o0 + h;
                src[h] = o < r_end ? (p.nbr ? __ldg(p.nbr + (long long)k * p.nbr_stride + o) : o) : -1;
            }
            const bool any = __any_sync(0xffffffffu, src[0] >= 0 || src[1] >= 0);     // every producer warp holds the same rows
            if (any) {
                unsigned char* st = gen + (size_t)s * stage_bytes;
                for (int cg = warp; cg < BM / 8; cg += 4) {          // A = X^T: input channels m0 + [0, 128)
                    float v0[8], v1[8];
                    load8(p.x, p.cin, src[0], m0 + cg * 8, 1.f, v0);
                    load8(p.x, p.cin, src[1], m0 + cg * 8, 1.f, v1);
                    store_pairs8(st, st + A_TILE, cg * 8, pr, v0, v1);
                }
                for (int cg = warp; cg < NC / 8; cg += 4) {          // B = G^T: output channels n0 + [0, NC); zero where X is absent
                    float v0[8], v1[8];
                    load8(p.g, p.cout, src[0] >= 0 ? o0 : -1, n0 + cg * 8, gs, v0);
                    load8(p.g, p.cout, src[1] >= 0 ? o0 + 1 : -1, n0 + cg * 8, gs, v1);
                    store_pairs8(st + 2u * A_TILE, st + 2u * A_TILE + b_tile, cg * 8, pr, v0, v1);
                }
            }
            if (threadIdx.x == 0) live[s] = any ? 1 : 0;
            fence_proxy_async();                 // generic-proxy stores, read by wgmma (async proxy)
            mbar_arrive(full(s));
        }
    } else {
        // =========================== consumers ===========================
        setmaxnreg_inc<CONSUMER_REGS>();
        const int wg = (warp >> 2) - 1;
        const bool active = m0 + wg * 64 < p.cin;          // a warpgroup whose 64 channels are all past cin only keeps the ring going
        float acc[NC / 2], tot[NC / 2];
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) tot[i] = 0.f;
        int in_group = 0, prev_s = -1;
        for (int i = 0; i < nst; ++i) {
            const int s = i % S;
            mbar_wait(full(s), (i / S) & 1);
            if (active && live[s]) {
                const uint32_t a_hi = base + (uint32_t)s * stage_bytes + (uint32_t)wg * (A_TILE / 2), a_lo = a_hi + A_TILE;
                const uint32_t b_hi = base + (uint32_t)s * stage_bytes + 2u * A_TILE, b_lo = b_hi + b_tile;
                reg_fence(acc);
                wg_stage_mma<NC>(acc, a_hi, a_lo, b_hi, b_lo, 4, in_group == 0);
                reg_fence(acc);
                wgmma_wait<1>();                             // the previous stage's MMAs are done: release it
                if (prev_s >= 0 && lane == 0) mbar_arrive(empty(prev_s));
                prev_s = s;
                if (++in_group == GROUP) {
                    wgmma_wait<0>();
                    reg_fence(acc);
                    if (lane == 0) mbar_arrive(empty(prev_s));
                    prev_s = -1;
#pragma unroll
                    for (int j = 0; j < NC / 2; ++j) tot[j] = __fadd_rn(tot[j], acc[j]);
                    in_group = 0;
                }
            } else {
                // an empty stage: release it, and the stage still held for its MMAs (the producer may next refill that very slot,
                // S stages on, before any further stage with MMAs comes to release it)
                if (prev_s >= 0) {
                    wgmma_wait<0>();
                    if (lane == 0) mbar_arrive(empty(prev_s));
                    prev_s = -1;
                }
                if (lane == 0) mbar_arrive(empty(s));
            }
        }
        if (in_group > 0) {
            wgmma_wait<0>();
            reg_fence(acc);
            // an empty stage after the group's last live one has already released it (prev_s = -1); empty(-1) would be the
            // address of full(MAX_STAGES - 1)
            if (prev_s >= 0 && lane == 0) mbar_arrive(empty(prev_s));
#pragma unroll
            for (int j = 0; j < NC / 2; ++j) tot[j] = __fadd_rn(tot[j], acc[j]);
        }
        wgmma_wait<0>();
        // register j of this thread: input channel row 16 (warp & 3) + lane / 4 + 8 ((j / 2) & 1), output channel 8 (j / 4) + 2 (lane & 3) + (j & 1)
        const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        float* dst = p.partial + ((long long)chunk * p.kvol + k) * p.cin * p.cout;
#pragma unroll
        for (int j = 0; j < NC / 2; j += 2) {
            const int m = r0 + 8 * ((j >> 1) & 1);
            const int n = n0 + 8 * (j >> 2) + 2 * (lane & 3);
            if (m < p.cin) *reinterpret_cast<float2*>(dst + (long long)m * p.cout + n) = make_float2(tot[j], tot[j + 1]);
        }
    }
}

// dw[i] = (sum over chunks c, ascending, of partial[c][i]) * 2^-k
__global__ void k_wgrad_reduce(const float* __restrict__ partial, int nchunks, long long total, const unsigned* __restrict__ header,
                               float* __restrict__ dw) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    float s = partial[i];
    for (int c = 1; c < nchunks; ++c) s = __fadd_rn(s, partial[(long long)c * total + i]);
    dw[i] = s * (1.f / weight_scale(*header));
}

static bool shape_ok(int kvol, int cin, int cout) {
    if (kvol != 1 && kvol != 8 && kvol != 27) return false;
    if (cin < 1 || cin > 512 || (cin % 8 != 0 && cin > 8)) return false;
    return cout == 32 || cout == 64 || cout == 96 || cout == 128 || cout == 256;
}

static size_t smem_bytes(int nc, int stages) {
    return 1024 + (size_t)stages * (2 * A_TILE + 2 * (size_t)nc * 128) + MAX_STAGES * sizeof(int) + 2 * MAX_STAGES * sizeof(uint64_t);
}

template <int NC>
static int launch(Lb2Handle* h, cudaStream_t s, Params p, int nchunks) {
    int stages = MAX_STAGES;
    while (stages > 2 && smem_bytes(NC, stages) > 227 * 1024) --stages;
    p.stages = stages;
    const size_t smem = smem_bytes(NC, stages);
    cudaError_t e = lb2_configure_smem(h, LB2_K_WGRAD + (NC / 32 - 1), k_spconv_wgrad<NC>, (int)(227 * 1024));
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "k_spconv_wgrad smem attribute: %s", cudaGetErrorString(e));
    const unsigned grid = (unsigned)((long long)nchunks * p.kvol * p.mblocks * p.nsplit);
    k_spconv_wgrad<NC><<<grid, THREADS, smem, s>>>(p);
    LB2_POST_LAUNCH(h, "k_spconv_wgrad");
    return LB2_OK;
}

}  // namespace wgrad
}  // namespace tc

extern "C" size_t lb2_spconv_wgrad_scratch_bytes(int32_t kvol, int32_t cin, int32_t cout, int32_t m_out) {
    if (!tc::wgrad::shape_ok(kvol, cin, cout) || m_out < 0) return 0;
    return tc::PACK_HEADER + (size_t)tc::wgrad::nchunks_of(m_out) * kvol * cin * cout * sizeof(float);
}

extern "C" int lb2_spconv_wgrad(void* handle, void* stream, const float* x, int32_t cin, const float* g, int32_t cout, int32_t m_out,
                                const int32_t* nbr, int64_t nbr_stride, int32_t kvol, float* dw, void* scratch) {
    using namespace tc::wgrad;
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && dw && scratch, "spconv_wgrad null");
    LB2_REQUIRE(h, m_out >= 0, "m_out");
    if (!shape_ok(kvol, cin, cout))
        return lb2_fail(h, LB2_ERR_UNSUP, "spconv_wgrad: no tensor-core kernel for this (kvol, cin, cout)%s", "");
    cudaStream_t s = (cudaStream_t)stream;
    const long long total = (long long)kvol * cin * cout;
    if (m_out == 0) {                    // no rows: G and the map are empty (an empty tensor may have no data pointer)
        if (cudaMemsetAsync(dw, 0, (size_t)total * sizeof(float), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "spconv_wgrad memset%s", "");
        return LB2_OK;
    }
    LB2_REQUIRE(h, x && g, "spconv_wgrad null");
    LB2_REQUIRE(h, nbr != nullptr || kvol == 1, "identity map only for kvol == 1");
    LB2_REQUIRE(h, nbr == nullptr || nbr_stride >= m_out, "nbr_stride");
    unsigned* header = (unsigned*)scratch;
    if (cudaMemsetAsync(header, 0, tc::PACK_HEADER, s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "spconv_wgrad memset%s", "");
    const long long ng = (long long)m_out * cout;
    tc::k_weight_absmax<<<(unsigned)std::min<long long>(cdiv(ng, 256), 1024), 256, 0, s>>>(g, ng, header);
    LB2_POST_LAUNCH(h, "k_weight_absmax");
    Params p;
    p.x = x; p.g = g; p.nbr = nbr; p.nbr_stride = nbr ? nbr_stride : 0;
    p.cin = cin; p.cout = cout; p.kvol = kvol; p.m_out = m_out;
    p.rows_per_chunk = rows_per_chunk_of(m_out);
    p.mblocks = (int)cdiv(cin, tc::BM);
    // at most 64 output channels per CTA: a consumer holds 32 accumulator and 32 total registers, and the producers stay within their
    // 88 registers without spilling (a 128-channel B gather does not)
    p.nsplit = cout % 64 == 0 ? cout / 64 : cout / 32;
    p.stages = 0;
    p.header = header;
    p.partial = reinterpret_cast<float*>((unsigned char*)scratch + tc::PACK_HEADER);
    const int nchunks = nchunks_of(m_out);
    int rc;
    if (cout / p.nsplit == 64) rc = launch<64>(h, s, p, nchunks);
    else rc = launch<32>(h, s, p, nchunks);
    if (rc != LB2_OK) return rc;
    k_wgrad_reduce<<<cdiv(total, 256), 256, 0, s>>>(p.partial, nchunks, total, header, dw);
    LB2_POST_LAUNCH(h, "k_wgrad_reduce");
    return LB2_OK;
}
