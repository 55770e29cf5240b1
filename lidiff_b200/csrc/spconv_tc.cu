// K4 (variant B) — sparse convolution as an output-stationary implicit GEMM on the Hopper tensor
// cores (wgmma, accumulator in registers), split-precision FP16x3 so that 49 stacked layers stay
// inside the 1e-3 fp32 parity bar:
//     x = x_hi + x_lo (fp16 each),  w*2^k = w_hi + w_lo,   x.w ~= (x_hi.w_hi + x_lo.w_hi + x_hi.w_lo) * 2^-k
// (22 mantissa bits per operand; the dropped x_lo.w_lo term is ~2^-22 relative.  BF16x3 costs the same
// three MMAs and is far less accurate.  Weights are pre-scaled by a power of two per layer so their low
// parts stay in fp16's normal range; activations saturate at +-65504.)
//
// One CTA owns 128 output rows x NC output channels (NC = Cout, or Cout / 2 for Cout > 128: blockIdx.z picks
// the half).  Warp roles (384 threads, three warpgroups):
//   warpgroup 0  producers: gather the neighbour rows of kernel offset k / channel chunk c (fp32 rows split to
//                fp16 hi/lo in registers, or the fp16 split companions with cp.async) into the K-major
//                SWIZZLE_128B shared-memory image; thread 0 also streams the pre-packed weight tiles of (k, c)
//                with cp.async.bulk (mbarrier complete_tx).
//   warpgroups 1, 2  consumers: rows [0, 64) / [64, 128) of the tile, 3 x (chunk / 16) wgmma per stage.
//                TWO-LEVEL ACCUMULATION: a long chain of tensor-core accumulations loses accuracy linearly with
//                its length, so the chain is cut into groups of <= STEP_BUDGET MMA steps, each started from zero;
//                after each group the partial sum is added to a running fp32 total in registers (round-to-nearest).
//                The totals go through a shared-memory staging tile to a coalesced epilogue:
//                BN affine + residual + ReLU + gate -> global.
// Kernel offsets where none of the tile's 128 rows has a neighbour are skipped by every role.
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
    int stages, nchunks, group;                         // group: kernel offsets per accumulation group
    lb2_conv_io io[2];
};

template <int NC>
__global__ void __launch_bounds__(THREADS, 1) k_spconv_tc(const Params p) {
    extern __shared__ unsigned char smem_raw[];
    const int M = p.d_mout ? min(*p.d_mout, p.mout_cap) : p.mout_cap;
    const int m0 = blockIdx.x * BM;
    if (m0 >= M) return;
    const lb2_conv_io io = p.io[blockIdx.y];
    const int n0 = blockIdx.z * NC;                  // first output channel of this CTA
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ctot = p.c1 + p.c2;

    // ---- shared memory carve-up (tiles 1024-byte aligned for SWIZZLE_128B) -----------------------------
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char* gen = smem_raw + (base - raw);
    constexpr uint32_t b_tile = (uint32_t)NC * 128u;                 // one fp16 B tile (hi or lo) of this CTA's channels
    const uint32_t b_full = (uint32_t)p.cout * 128u;                 // the same tile over all cout channels (packed layout)
    const uint32_t stage_bytes = 2u * A_TILE + 2u * b_tile;
    unsigned char* tail = gen + (size_t)p.stages * stage_bytes;
    int* idx_s = reinterpret_cast<int*>(tail);                       // [kvol][BM]
    uint64_t* bars = reinterpret_cast<uint64_t*>(tail + MAX_KVOL * BM * sizeof(int));
    uint32_t* misc = reinterpret_cast<uint32_t*>(bars + 3 * MAX_STAGES);      // [1] offset mask
    int* row_s = reinterpret_cast<int*>(misc + 4);                             // [BM] output row of each tile slot
    const uint32_t bar0 = smem_u32(bars);
    auto full_a = [&](int s) { return bar0 + 8u * s; };
    auto full_b = [&](int s) { return bar0 + 8u * (MAX_STAGES + s); };
    auto empty = [&](int s) { return bar0 + 8u * (2 * MAX_STAGES + s); };

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(full_a(s), NUM_PRODUCER); mbar_init(full_b(s), 1); mbar_init(empty(s), NUM_CONSUMER_WARPS); }
        misc[1] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // ---- neighbour indices of this tile + mask of non-empty kernel offsets -----------------------------
    if (threadIdx.x < BM) {
        const int slot = m0 + threadIdx.x;
        const int row = (slot < M) ? (p.row_perm ? __ldg(p.row_perm + slot) : slot) : -1;
        row_s[threadIdx.x] = row;
        uint32_t mymask = 0;
        for (int k0 = 0; k0 < p.kvol; k0 += 9) {        // 9 independent loads in flight, then the votes
            int v[9];
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                const int k = k0 + q;
                v[q] = -1;
                if (k < p.kvol && row >= 0) v[q] = p.nbr ? __ldg(p.nbr + (long long)k * p.nbr_stride + row) : row;
            }
#pragma unroll
            for (int q = 0; q < 9; ++q) {
                const int k = k0 + q;
                if (k < p.kvol) {
                    idx_s[k * BM + threadIdx.x] = v[q];
                    if (__any_sync(0xffffffffu, v[q] >= 0)) mymask |= 1u << k;
                }
            }
        }
        if (lane == 0 && mymask) atomicOr(&misc[1], mymask);
    }
    __syncthreads();
    const uint32_t kmask = misc[1];
    const int n_off = __popc(kmask);

    if (warp < 4) {
        // =========================== producers: A gather (all 128 threads), B weights (thread 0) ===========================
        const int sub = threadIdx.x & 7;           // 8-channel group inside the 64-channel chunk
        const int rbase = threadIdx.x >> 3;        // 0..15
        const bool use_h = (io.in1_h != nullptr) && (p.c2 == 0 || io.in2_h != nullptr);   // fp16 split inputs: cp.async gather
        // cp.async lookahead: stages still landing while the next is issued.  S - 2, not S - 1: a consumer releases a stage only once it
        // holds the next one (wgmma_wait<1>), so the producers must be able to publish stage i + 1 while stage i - 1 is still held
        const int D = max(p.stages - 2, 0);
        int it = 0, arrived = 0;
        for (uint32_t km = kmask; km; km &= km - 1) {
            const int k = __ffs(km) - 1;
            const int* idxk = idx_s + k * BM;
            int src[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) src[j] = idxk[rbase + 16 * j];
            for (int c = 0; c < p.nchunks; ++c, ++it) {
                const int s = it % p.stages;
                mbar_wait(empty(s), ((it / p.stages) & 1) ^ 1);
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
                if (use_h) {
                    cp_async_commit();
                    if (it >= D) {                 // the copies of iteration it-D have landed
                        cp_async_wait_dyn(D);
                        fence_proxy_async();
                        mbar_arrive(full_a(arrived % p.stages));
                        ++arrived;
                    }
                } else {
                    fence_proxy_async();
                    mbar_arrive(full_a(s));
                }
            }
        }
        if (use_h) {
            cp_async_wait<0>();
            fence_proxy_async();
            for (; arrived < it; ++arrived) mbar_arrive(full_a(arrived % p.stages));
        }
    } else {
        // =========================== consumers: wgmma + two-level accumulation ===========================
        const int wg = (warp >> 2) - 1;                           // 0: tile rows [0, 64), 1: rows [64, 128)
        float acc[NC / 2], tot[NC / 2];
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) tot[i] = 0.f;
        int it = 0, in_group = 0, off_idx = 0, prev_s = -1;
        bool have_tot = false;
        for (uint32_t km = kmask; km; km &= km - 1, ++off_idx) {
            for (int c = 0; c < p.nchunks; ++c, ++it) {
                const int s = it % p.stages;
                const uint32_t par = (it / p.stages) & 1;
                mbar_wait(full_b(s), par);
                mbar_wait(full_a(s), par);
                const uint32_t a_hi = base + (uint32_t)s * stage_bytes + (uint32_t)wg * (A_TILE / 2), a_lo = a_hi + A_TILE;
                const uint32_t b_hi = base + (uint32_t)s * stage_bytes + 2u * A_TILE, b_lo = b_hi + b_tile;
                const int ksteps = min(KC, ctot - c * KC) >> 4;
                reg_fence(acc);
                wg_stage_mma<NC>(acc, a_hi, a_lo, b_hi, b_lo, ksteps, in_group == 0 && c == 0);   // first MMA of a group overwrites
                reg_fence(acc);
                wgmma_wait<1>();                                  // the MMAs of the previous stage are done: release it
                if (prev_s >= 0 && lane == 0) mbar_arrive(empty(prev_s));
                prev_s = s;
            }
            if (++in_group == p.group || off_idx == n_off - 1) {  // partial sum of this group complete -> running total
                wgmma_wait<0>();
                reg_fence(acc);
                if (lane == 0) mbar_arrive(empty(prev_s));
                prev_s = -1;
#pragma unroll
                for (int i = 0; i < NC / 2; ++i) tot[i] = have_tot ? __fadd_rn(tot[i], acc[i]) : acc[i];
                have_tot = true;
                in_group = 0;
            }
        }
        // ---- totals -> shared-memory staging tile (the stage ring is idle once both consumer warpgroups are here) ----------
        const float out_scale = __ldg(reinterpret_cast<const float*>(p.wpacked) + 1);     // 2^-k of the packed weights
        float* stage_c = reinterpret_cast<float*>(gen);            // [BM][pitch] fp32
        constexpr int pitch = NC + 4;                              // +4 floats: fewer bank conflicts on the row reads
        asm volatile("bar.sync 1, 256;" ::: "memory");
        {
            const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
            for (int i = 0; i < NC / 2; i += 2) {
                const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3);
                *reinterpret_cast<float2*>(stage_c + row * pitch + col) = make_float2(tot[i] * out_scale, tot[i + 1] * out_scale);
            }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        // ---- epilogue, coalesced: consumer warp cw owns tile rows cw, cw + 8, ... and walks their (row, 4-channel) elements with
        //      consecutive lanes on consecutive channels, so every global access is a contiguous row segment ----------
        const int cw = warp - 4;
        constexpr int nv = NC >> 2;                                // float4 per row (this CTA's channels)
        for (int e = lane; e < (BM / NUM_CONSUMER_WARPS) * nv; e += 32) {
            const int rr = cw + NUM_CONSUMER_WARPS * (e / nv);
            const int lcol = (e % nv) * 4;
            const int col = n0 + lcol;
            const int orow = row_s[rr];
            if (orow < 0) continue;
            const long long ro = (long long)orow * p.cout;
            const float4 a4 = *reinterpret_cast<const float4*>(stage_c + (size_t)rr * pitch + lcol);
            float y[4] = {a4.x, a4.y, a4.z, a4.w};
            if (io.pre_add) {
                const float4 t4 = __ldg(reinterpret_cast<const float4*>(io.pre_add + ro + col));
                y[0] += t4.x; y[1] += t4.y; y[2] += t4.z; y[3] += t4.w;
            }
            if (p.scale) {
                const float4 s4 = __ldg(reinterpret_cast<const float4*>(p.scale + col));
                const float4 h4 = __ldg(reinterpret_cast<const float4*>(p.shift + col));
                y[0] = fmaf(y[0], s4.x, h4.x); y[1] = fmaf(y[1], s4.y, h4.y); y[2] = fmaf(y[2], s4.z, h4.z); y[3] = fmaf(y[3], s4.w, h4.w);
            }
            if (io.residual || io.residual_h) {
                const float4 t4 = load_residual4(io.residual, io.residual_h, orow, p.cout, col);
                y[0] += t4.x; y[1] += t4.y; y[2] += t4.z; y[3] += t4.w;
            }
            if (p.relu) {
#pragma unroll
                for (int j = 0; j < 4; ++j) y[j] = fmaxf(y[j], 0.f);
            }
            if (io.out) *reinterpret_cast<float4*>(io.out + ro + col) = make_float4(y[0], y[1], y[2], y[3]);
            if (io.out_h) store_split4(io.out_h, orow, p.cout, col, y);
            if (io.out_gated || io.out_gated_h) {
                if (io.gate_table) {
                    const long long g = io.gate_idx ? __ldg(io.gate_idx + orow) : 0;
                    const float4 g4 = __ldg(reinterpret_cast<const float4*>(io.gate_table + g * p.cout + col));
                    y[0] *= g4.x; y[1] *= g4.y; y[2] *= g4.z; y[3] *= g4.w;
                }
                if (io.out_gated) *reinterpret_cast<float4*>(io.out_gated + ro + col) = make_float4(y[0], y[1], y[2], y[3]);
                if (io.out_gated_h) store_split4(io.out_gated_h, orow, p.cout, col, y);
            }
        }
    }
}

// ---- weight packing: (kvol, cin, cout) fp32 -> [256 B header][per (k, chunk): hi tile | lo tile], each tile cout rows
// x 128 B in the K-major SWIZZLE_128B image, channels beyond cin zero-filled.  Values are W * 2^k with k chosen so
// that max|W| * 2^k lies in [8192, 16384); header[1] = 2^-k is applied to the accumulator in the epilogue. ---------
__global__ void k_weight_absmax(const float* __restrict__ w, long long n, unsigned* __restrict__ header) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float m = 0.f;
    for (; t < n; t += (long long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[t]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(header, __float_as_uint(m));      // non-negative floats order like uints
}

__device__ __forceinline__ float weight_scale(unsigned max_bits) {
    const float m = __uint_as_float(max_bits);
    if (!(m > 0.f) || !isfinite(m)) return 1.f;
    int e;
    frexpf(m, &e);                         // m = f * 2^e, f in [0.5, 1)
    return ldexpf(1.f, 14 - e);            // m * scale in [8192, 16384)
}

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
    return 1024 + (size_t)stages * (2 * A_TILE + 2 * (size_t)nc * 128) + MAX_KVOL * BM * sizeof(int) + 3 * MAX_STAGES * 8 + 16 + BM * sizeof(int);
}

template <int NC>
static int launch(Lb2Handle* h, cudaStream_t s, const Params& p, int npass, int nsplit, int stages) {
    const size_t smem = smem_bytes(NC, stages);
    cudaError_t e = lb2_configure_smem(h, LB2_K_TC + (NC / 32 - 1), k_spconv_tc<NC>, (int)(227 * 1024));
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "k_spconv_tc smem attribute: %s", cudaGetErrorString(e));
    dim3 grid(cdiv(p.mout_cap, BM), npass, nsplit);
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
    p.nchunks = (d->c1 + d->c2 + tc::KC - 1) / tc::KC;
    // a consumer thread holds NC / 2 accumulator and NC / 2 total registers: NC <= 128, so Cout 256 runs as two CTAs of 128 channels
    const int nsplit = d->cout > 128 ? 2 : 1;
    const int nc = d->cout / nsplit;
    int stages = tc::MAX_STAGES;
    while (stages > 2 && tc::smem_bytes(nc, stages) > 227 * 1024) --stages;
    p.stages = stages;
    const int steps_per_offset = 3 * ((d->c1 + d->c2 + 15) / 16);
    p.group = std::max(1, tc::STEP_BUDGET / steps_per_offset);
    p.io[0] = d->io[0]; p.io[1] = d->io[d->npass > 1 ? 1 : 0];
    switch (nc) {
        case 32: return tc::launch<32>(h, s, p, d->npass, nsplit, stages);
        case 64: return tc::launch<64>(h, s, p, d->npass, nsplit, stages);
        case 96: return tc::launch<96>(h, s, p, d->npass, nsplit, stages);
        case 128: return tc::launch<128>(h, s, p, d->npass, nsplit, stages);
        default: return lb2_fail(h, LB2_ERR_UNSUP, "tensor-core variant: no kernel for %s output channels per CTA", nc == 80 ? "80" : nc == 112 ? "112" : "this many");
    }
}
