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
__device__ __forceinline__ void wgmma_m64n96(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_m64n128(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate) : "memory");
}

// D(64 x N) for N = 32 / 64 / 96 / 128 as ONE instruction: every B row (= output channel) of the tile in one MMA, so each A slice is
// read from shared memory once per (A, B) pair.  The register layout above holds for any N, so D is the same array as before.
template <int N>
__device__ __forceinline__ void wgmma_n(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 32 || N == 64 || N == 96 || N == 128, "wgmma_n: N must be 32, 64, 96 or 128");
    if constexpr (N == 128) wgmma_m64n128(d, da, db, accumulate);
    else if constexpr (N == 96) wgmma_m64n96(d, da, db, accumulate);
    else if constexpr (N == 64) wgmma_m64n64(d, da, db, accumulate);
    else wgmma_m64n32(d, da, db, accumulate);
}
template <int N, int KSTEPS>
__device__ __forceinline__ void wg_stage_mma_k(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, uint32_t acc0) {
    wgmma_fence();          // in the MMAs' own basic block: a fence behind a branch makes ptxas inject warpgroup.arrive (C7519)
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
        const uint64_t dah = make_desc(a_hi + ks * 32), dal = make_desc(a_lo + ks * 32);
        const uint64_t dbh = make_desc(b_hi + ks * 32), dbl = make_desc(b_lo + ks * 32);
        wgmma_n<N>(d, dah, dbh, ks == 0 ? acc0 : 1u);
        wgmma_n<N>(d, dal, dbh, 1u);
        wgmma_n<N>(d, dah, dbl, 1u);
    }
    wgmma_commit();
}
// one pipeline stage of the FP16x3 product for the calling warpgroup: rows [64 wg, +64) of the A tiles (hi, lo) times the N rows of
// the B tiles (hi, lo), ksteps 16-channel steps, 3 MMAs each (x_hi.w_hi + x_lo.w_hi + x_hi.w_lo); first = overwrite D.
// ksteps is 4 except in the last chunk of a channel count that is not a multiple of 64 (channel counts are multiples of 16): every
// case is a fully unrolled instruction sequence, so no loop counter or accumulator copy sits between the MMAs of a stage.
template <int N>
__device__ __forceinline__ void wg_stage_mma(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, int ksteps, bool first) {
    const uint32_t acc0 = first ? 0u : 1u;
    if (ksteps == 4) wg_stage_mma_k<N, 4>(d, a_hi, a_lo, b_hi, b_lo, acc0);
    else if (ksteps == 2) wg_stage_mma_k<N, 2>(d, a_hi, a_lo, b_hi, b_lo, acc0);
    else if (ksteps == 1) wg_stage_mma_k<N, 1>(d, a_hi, a_lo, b_hi, b_lo, acc0);
    else wg_stage_mma_k<N, 3>(d, a_hi, a_lo, b_hi, b_lo, acc0);
}
// role of the calling thread's warpgroup (threadIdx.x / 128), read from lane 0 so that the compiler sees a warp-uniform value: a
// branch on threadIdx.x itself counts as divergent, and ptxas then serialises every wgmma behind it (C7520)
__device__ __forceinline__ int warpgroup_role() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0); }
// hand registers from the producer warpgroup to the consumer warpgroups (the CTA's register file is fixed at launch)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {      // keeps the compiler from moving accumulator accesses across a wgmma wait
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// byte offset of (row, 16-byte chunk) inside a K-major SWIZZLE_128B tile (rows of 128 B, Swizzle<3,4,3>)
__device__ __forceinline__ uint32_t sw128(int row, int chunk) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

// RN_sat: fp32 -> fp16 rounded to nearest-even, results beyond the fp16 range (infinities included) clamped to +-65504, NaN kept NaN
// (cvt .satfinite); RN: the same rounding without the clamp (beyond 65504 -> +-inf).  Two values at once, x in the low half.
__device__ __forceinline__ uint32_t cvt_f16x2_sat(float x, float y) {
    uint32_t d;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(y), "f"(x));
    return d;
}
__device__ __forceinline__ uint32_t cvt_f16x2_rn(float x, float y) {
    uint32_t d;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(y), "f"(x));
    return d;
}
// THE fp32 -> fp16 (hi, lo) split of the FP16x3 product: every split companion (conv epilogues, gate_mul) and every A-operand image
// gathered from fp32 rows is written by it, so a result does not depend on which kernel produced its input or how it was gathered.
//   hi = RN_sat(x),  lo = RN(x - hi).
//   |x| < 131024: hi + lo = x to 2^-22 relative; below |x| = 2^-3 lo is an fp16 subnormal, so the error has an absolute floor of
//   2^-25 (|x| < 2^-25 splits to zero).  Beyond 65504 hi saturates and lo carries the rest.
//   |x| >= 131024, +-inf included: lo = +-inf, so every product that reads x is non-finite, as in the fp32 convolutions.
//   NaN: hi = lo = NaN.
// Two values per call: x0 in the low halves of hi and lo, x1 in the high halves.
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    hi = cvt_f16x2_sat(x0, x1);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = cvt_f16x2_rn(x0 - f.x, x1 - f.y);
}
__device__ __forceinline__ void split1(float x, __half& hi, __half& lo) {
    uint32_t h, l;
    split2(x, 0.f, h, l);
    hi = __ushort_as_half((unsigned short)(h & 0xFFFFu));
    lo = __ushort_as_half((unsigned short)(l & 0xFFFFu));
}
__device__ __forceinline__ void split8(const float4& a, const float4& b, uint4& hi, uint4& lo) {
    split2(a.x, a.y, hi.x, lo.x);
    split2(a.z, a.w, hi.y, lo.y);
    split2(b.x, b.y, hi.z, lo.z);
    split2(b.z, b.w, hi.w, lo.w);
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

// power-of-two pre-scale of the operand that the FP16x3 product splits like a weight (the packed weights of the forward, the output
// gradient of the weight gradient): header[0] = max|v| over the finite v as float bits (atomicMax, the caller zeroes it first), and
// v * weight_scale(header[0]) has its largest finite magnitude in [8192, 16384).  A NaN or +-inf element is skipped: it makes the
// outputs that read it non-finite whatever the scale, and taking its magnitude (fmaxf skips NaN, but +inf wins) would leave every
// other element unscaled, its low half lost below the fp16 subnormal range.
static __global__ void k_weight_absmax(const float* __restrict__ w, long long n, unsigned* __restrict__ header) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float m = 0.f;
    for (; t < n; t += (long long)gridDim.x * blockDim.x) {
        const float a = fabsf(w[t]);
        if (isfinite(a)) m = fmaxf(m, a);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(header, __float_as_uint(m));      // non-negative floats order like uints
}

__device__ __forceinline__ float weight_scale(unsigned max_bits) {
    const float m = __uint_as_float(max_bits);
    if (!(m > 0.f) || !isfinite(m)) return 1.f;
    int e;
    frexpf(m, &e);                         // m = f * 2^e, f in [0.5, 1)
    // m * scale in [8192, 16384); below m = 2^-113 it stops at 2^126, so that the scale and header[1] = 2^-126 stay finite, nonzero
    // and normal (nothing depends on how the build treats fp32 subnormals)
    return ldexpf(1.f, min(14 - e, 126));
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
