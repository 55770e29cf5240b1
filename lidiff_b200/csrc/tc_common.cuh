// Device helpers shared by the wgmma kernels (spconv_tc.cu, spconv_scatter.cu): mbarrier / bulk-TMA / wgmma
// PTX wrappers, GMMA shared-memory descriptors, the K-major SWIZZLE_128B addressing and the fp32 -> fp16 hi/lo split.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace tc {

constexpr int BM = 128;              // rows per tile (two consumer warpgroups of wgmma M = 64)
constexpr int KC = 64;               // channels per pipeline stage (one 128-byte swizzle atom of fp16)
constexpr int A_TILE = BM * KC * 2;  // bytes of one fp16 A tile (hi or lo): 16 KB
constexpr int PACK_HEADER = 256;     // packed weights: [0] max|W| bits, [1] 2^-k output scale

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// try_wait with a suspend-time hint (as CUTLASS' ClusterBarrier::wait): the thread sleeps in hardware until the phase completes or the
// hint expires instead of spinning through the loop — waiting warps no longer take issue slots from the working warps of their
// scheduler (ncu on the sparse levels' layers: 14 % of all executed instructions were wait loops).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity), "r"(0x989680u) : "memory");
    }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// K-major SWIZZLE_128B shared-memory matrix descriptor of wgmma (cute::GMMA::GmmaDescriptor):
//   [0,14) start>>4 | [16,30) LBO>>4 (=1, unused for swizzled K-major) | [32,46) SBO>>4 (8 rows x 128 B = 1024 B)
//   [49,52) base offset = 0 (tiles are 1024-byte aligned) | [62,64) layout = 1 (SWIZZLE_128B)
// A step of 16 channels inside the 128-byte swizzle atom advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D(64 x n, fp32 registers) (+)= A(64 x 16, smem) . B(n x 16, smem)^T, both operands fp16 K-major.  accumulate = 0 overwrites D.
// Register i of the calling thread (warp w, lane l of the warpgroup) holds row 16 w + l / 4 + 8 ((i / 2) & 1),
// column 8 (i / 4) + 2 (l % 4) + (i & 1).
__device__ __forceinline__ void wgmma_m64n16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_m64n32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_m64n64(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate) : "memory");
}

// D(64 x N) for N a multiple of 16: n64 / n32 / n16 instructions side by side, B rows (= output channels) advance 128 bytes each
template <int N, int OFF = 0>
__device__ __forceinline__ void wgmma_n(float (&d)[N / 2], uint64_t da, uint32_t b_addr, uint32_t accumulate) {
    constexpr int REST = N - OFF;
    if constexpr (REST >= 64) {
        wgmma_m64n64(d + OFF / 2, da, make_desc(b_addr + OFF * 128), accumulate);
        wgmma_n<N, OFF + 64>(d, da, b_addr, accumulate);
    } else if constexpr (REST >= 32) {
        wgmma_m64n32(d + OFF / 2, da, make_desc(b_addr + OFF * 128), accumulate);
        wgmma_n<N, OFF + 32>(d, da, b_addr, accumulate);
    } else if constexpr (REST >= 16) {
        wgmma_m64n16(d + OFF / 2, da, make_desc(b_addr + OFF * 128), accumulate);
    }
}
// one pipeline stage of the FP16x3 product for the calling warpgroup: rows [64 wg, +64) of the A tiles (hi, lo) times the N rows of
// the B tiles (hi, lo), ksteps 16-channel steps, 3 MMAs each (x_hi.w_hi + x_lo.w_hi + x_hi.w_lo); first = overwrite D
template <int N>
__device__ __forceinline__ void wg_stage_mma(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, int ksteps, bool first) {
    wgmma_fence();
#pragma unroll 1
    for (int ks = 0; ks < ksteps; ++ks) {
        const uint64_t dah = make_desc(a_hi + ks * 32), dal = make_desc(a_lo + ks * 32);
        wgmma_n<N>(d, dah, b_hi + ks * 32, (first && ks == 0) ? 0u : 1u);
        wgmma_n<N>(d, dal, b_hi + ks * 32, 1u);
        wgmma_n<N>(d, dah, b_lo + ks * 32, 1u);
    }
    wgmma_commit();
}
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {      // keeps the compiler from moving accumulator accesses across a wgmma wait
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// byte offset of (row, 16-byte chunk) inside a K-major SWIZZLE_128B tile (rows of 128 B, Swizzle<3,4,3>)
__device__ __forceinline__ uint32_t sw128(int row, int chunk) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

// two fp32 -> packed (hi, hi) and (lo, lo) fp16 pairs.  F2FP.SATFINITE rounds each half independently to nearest-even and clamps to
// +-65504 instead of producing inf, so inside the fp16 range the results equal the scalar split1 below bit for bit (beyond it hi
// saturates and lo carries what it can of the rest)
__device__ __forceinline__ uint32_t cvt_f16x2_sat(float lo_half, float hi_half) {
    uint32_t d;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi_half), "f"(lo_half));
    return d;
}
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    hi = cvt_f16x2_sat(x0, x1);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = cvt_f16x2_sat(x0 - f.x, x1 - f.y);
}
__device__ __forceinline__ void split8(const float4& a, const float4& b, uint4& hi, uint4& lo) {
    split2(a.x, a.y, hi.x, lo.x);
    split2(a.z, a.w, hi.y, lo.y);
    split2(b.x, b.y, hi.z, lo.z);
    split2(b.z, b.w, hi.w, lo.w);
}


// fp32 -> (hi, lo) fp16 pair, saturating at the fp16 range
__device__ __forceinline__ void split1(float x, __half& hi, __half& lo) {
    x = fminf(fmaxf(x, -65504.f), 65504.f);
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}
// write 4 consecutive channels of a split companion row: hi halfs at row[col], lo halfs at row[c + col]
__device__ __forceinline__ void store_split4(void* base, long long row, int c, int col, const float (&y)[4]) {
    __half* rp = reinterpret_cast<__half*>(base) + row * 2 * c;
    uint2 uh, ul;
    split2(y[0], y[1], uh.x, ul.x);
    split2(y[2], y[3], uh.y, ul.y);
    *reinterpret_cast<uint2*>(rp + col) = uh;
    *reinterpret_cast<uint2*>(rp + c + col) = ul;
}
// 4 consecutive channels of a residual row: from the fp32 tensor, else from its split companion (hi + lo), else zero
__device__ __forceinline__ float4 load_residual4(const float* res, const void* res_h, long long row, int c, int col) {
    if (res) return __ldg(reinterpret_cast<const float4*>(res + row * c + col));
    if (!res_h) return make_float4(0.f, 0.f, 0.f, 0.f);
    const __half* rp = reinterpret_cast<const __half*>(res_h) + row * 2 * c + col;
    const uint2 uh = __ldg(reinterpret_cast<const uint2*>(rp)), ul = __ldg(reinterpret_cast<const uint2*>(rp + c));
    const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&uh.x)), h1 = __half22float2(*reinterpret_cast<const __half2*>(&uh.y));
    const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&ul.x)), l1 = __half22float2(*reinterpret_cast<const __half2*>(&ul.y));
    return make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_wait_dyn(int n) {      // n in [0, 3]
    if (n <= 0) cp_async_wait<0>(); else if (n == 1) cp_async_wait<1>(); else if (n == 2) cp_async_wait<2>(); else cp_async_wait<3>();
}

// One producer thread's share of an A stage (8 rows x one 8-channel group, hi and lo tile).
//  * split path  (src_h != nullptr): two 16-byte cp.async per row straight into the swizzled image (zero-fill for
//    missing rows); completion is tracked by the caller with commit/wait groups;
//  * fp32 path: 2 x LDG.128 per row, hi/lo split in registers, 2 x STS.128.
__device__ __forceinline__ void produce_a_split(const __half* __restrict__ src_h, int cw, int co, const int (&src)[8],
                                                uint32_t a_hi, uint32_t a_lo, int rbase, int sub) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint32_t off = sw128(rbase + 16 * j, sub);
        const bool ok = src[j] >= 0;
        const __half* rp = src_h + (ok ? ((long long)src[j] * 2 * cw + co) : 0);
        cp_async16(a_hi + off, rp, ok ? 16u : 0u);
        cp_async16(a_lo + off, rp + (ok ? cw : 0), ok ? 16u : 0u);
    }
}
__device__ __forceinline__ void produce_a_f32(const float* __restrict__ srcp, int cw, int co, const int (&src)[8],
                                              unsigned char* a_hi, unsigned char* a_lo, int rbase, int sub) {
    float4 va[8], vb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (src[j] >= 0) {
            const float4* rp = reinterpret_cast<const float4*>(srcp + (long long)src[j] * cw + co);
            va[j] = __ldg(rp);
            vb[j] = __ldg(rp + 1);
        } else {
            va[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            vb[j] = va[j];
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        uint4 hi, lo;
        split8(va[j], vb[j], hi, lo);
        const uint32_t off = sw128(rbase + 16 * j, sub);
        *reinterpret_cast<uint4*>(a_hi + off) = hi;
        *reinterpret_cast<uint4*>(a_lo + off) = lo;
    }
}

}  // namespace tc
