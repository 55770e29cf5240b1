// lb2_segment_dot: out[s] = sum over i in [offsets[s], offsets[s + 1]) of a[order[i]] * b[order[i]] (element-wise; b NULL: of a[order[i]]),
// the gradient of the conditioning gates' row gather (x * table[idx]: d table[j] = sum over the rows with idx = j of G * x).
//
// A few thousand segments share 10^5 - 10^6 rows, and in the unconditional training step one segment holds every row of its scan, so
// the work items are fixed-size chunks of the row order, not segments: chunk k is the positions [k R, (k + 1) R) whatever segments they
// belong to, one warp per chunk.  A chunk's run of positions inside one segment is a piece.  A segment that lies inside one chunk
// is written to `out` by that chunk's warp; a segment that crosses a chunk boundary has one piece per chunk it touches, each written
// to scratch, and k_segment_dot_reduce adds them in ascending chunk order.  No float atomics: the same bits on every run.
#include "common.cuh"

namespace segdot {

constexpr int R = LB2_SEGMENT_DOT_R;
constexpr int WARPS = 8;                // chunks per CTA
static_assert(R % 32 == 0 && R >= 32, "the row order of a chunk is staged as R / 32 registers per lane");

__device__ __forceinline__ float4 mul_rn(float4 p, float4 q) {
    return make_float4(__fmul_rn(p.x, q.x), __fmul_rn(p.y, q.y), __fmul_rn(p.z, q.z), __fmul_rn(p.w, q.w));
}
__device__ __forceinline__ float mul_rn(float p, float q) { return __fmul_rn(p, q); }
__device__ __forceinline__ float4 add_rn(float4 p, float4 q) {
    return make_float4(__fadd_rn(p.x, q.x), __fadd_rn(p.y, q.y), __fadd_rn(p.z, q.z), __fadd_rn(p.w, q.w));
}
__device__ __forceinline__ float add_rn(float p, float q) { return __fadd_rn(p, q); }
__device__ __forceinline__ void zero(float4& v) { v = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void zero(float& v) { v = 0.f; }

// V = float4: a lane owns 4 consecutive channels (c % 4 == 0, 16-byte loads); V = float: one channel.  Lanes run over the channel
// groups, 32 at a time; the chunk is walked once per 32 groups (one walk for c <= 128 on the vector path).
template <class V, bool MUL>
__global__ void __launch_bounds__(WARPS * 32, 2) k_segment_dot_chunks(const V* __restrict__ a, const V* __restrict__ b,
                                                                   const int64_t* __restrict__ order, const int64_t* __restrict__ offsets,
                                                                   int64_t nseg, int64_t nrows, int cv, V* __restrict__ partial,
                                                                   V* __restrict__ out) {
    // rows whose loads are issued before the first of them is added: 128 bytes per lane in flight with both operands
    constexpr int UNROLL = MUL && sizeof(V) == 16 ? 4 : 8;
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * WARPS + (threadIdx.x >> 5);
    const int64_t cb = k * R;
    if (cb >= nrows) return;
    const int64_t ce = min(cb + R, nrows);
    // the chunk's row indices, read coalesced: position cb + 32 j + l sits in register j of lane l
    int64_t ord[R / 32];
#pragma unroll
    for (int j = 0; j < R / 32; ++j) {
        const int64_t pos = cb + 32 * j + lane;
        ord[j] = pos < ce ? (order ? __ldg(order + pos) : pos) : 0;
    }
    // the segment that holds position cb: offsets[s0] <= cb < offsets[s0 + 1] (offsets[0] = 0 and offsets[nseg] = nrows)
    int64_t s0 = 0, hi = nseg;
    while (hi - s0 > 1) {
        const int64_t mid = (s0 + hi) >> 1;
        if (__ldg(offsets + mid) <= cb) s0 = mid; else hi = mid;
    }
    for (int v0 = 0; v0 < cv; v0 += 32) {
        const int v = v0 + lane;
        const bool live = v < cv;
        int64_t seg = s0, pb = cb;
        while (pb < ce) {
            const int64_t sb = __ldg(offsets + seg), se = __ldg(offsets + seg + 1);
            const int64_t pe = min(se, ce);
            const int l0 = (int)(pb - cb), l1 = (int)(pe - cb);
            V acc;
            zero(acc);
#pragma unroll
            for (int j = 0; j < R / 32; ++j) {
                const int lo = max(l0, 32 * j) - 32 * j, up = min(l1, 32 * j + 32) - 32 * j;
                int u = lo;
                for (; u + UNROLL <= up; u += UNROLL) {
                    V p[UNROLL], q[UNROLL];
#pragma unroll
                    for (int t = 0; t < UNROLL; ++t) {
                        const int64_t row = __shfl_sync(0xffffffffu, ord[j], u + t);
                        if (live) {
                            p[t] = __ldg(a + row * cv + v);
                            if (MUL) q[t] = __ldg(b + row * cv + v);
                        }
                    }
                    if (live) {
#pragma unroll
                        for (int t = 0; t < UNROLL; ++t) acc = add_rn(acc, MUL ? mul_rn(p[t], q[t]) : p[t]);
                    }
                }
                for (; u < up; ++u) {
                    const int64_t row = __shfl_sync(0xffffffffu, ord[j], u);
                    if (live) {
                        const V p = __ldg(a + row * cv + v);
                        acc = add_rn(acc, MUL ? mul_rn(p, __ldg(b + row * cv + v)) : p);
                    }
                }
            }
            if (live) {
                if (sb >= cb && se <= ce) out[seg * cv + v] = acc;                       // the whole segment
                else partial[(2 * k + (pb != cb)) * cv + v] = acc;                     // slot 0: the piece that starts the chunk
            }
            pb = pe;
            if (pb < ce) {                                                              // the next segment with a row (pb < nrows)
                do ++seg; while (__ldg(offsets + seg + 1) <= pb);
            }
        }
    }
}

// segments without rows: zeros; segments inside one chunk: already written; the others: their pieces in ascending chunk order
__global__ void k_segment_dot_reduce(const int64_t* __restrict__ offsets, int64_t nseg, int c, const float* __restrict__ partial,
                                     float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nseg * c) return;
    const int64_t seg = i / c;
    const int j = (int)(i - seg * c);
    const int64_t sb = __ldg(offsets + seg), se = __ldg(offsets + seg + 1);
    if (sb >= se) { out[i] = 0.f; return; }
    const int64_t kb = sb / R, ke = (se - 1) / R;
    if (kb == ke) return;
    float s = __fadd_rn(0.f, partial[(2 * kb + (sb != kb * R)) * c + j]);
#pragma unroll 8
    for (int64_t k = kb + 1; k <= ke; ++k) s = __fadd_rn(s, partial[2 * k * c + j]);
    out[i] = s;
}

template <class V, bool MUL>
static void launch(cudaStream_t s, const float* a, const float* b, const int64_t* order, const int64_t* offsets, int64_t nseg,
                   int64_t nrows, int cv, float* partial, float* out) {
    k_segment_dot_chunks<V, MUL><<<cdiv(cdiv(nrows, R), WARPS), WARPS * 32, 0, s>>>((const V*)a, (const V*)b, order, offsets, nseg, nrows,
                                                                                  cv, (V*)partial, (V*)out);
}

}  // namespace segdot

extern "C" size_t lb2_segment_dot_scratch_bytes(int64_t nrows, int32_t c) {
    if (nrows < 0 || c < 1 || c > 256) return 0;
    return (size_t)(nrows / segdot::R + 1) * 2 * c * sizeof(float);
}

extern "C" int lb2_segment_dot(void* handle, void* stream, const float* a, const float* b, const int64_t* order, const int64_t* offsets,
                               int64_t nrows, int64_t nseg, int32_t c, float* out, void* scratch) {
    using namespace segdot;
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && nrows >= 0 && nseg >= 0, "segment_dot");
    LB2_REQUIRE(h, c >= 1 && c <= 256, "segment_dot: 1 <= c <= 256");
    if (nseg == 0) return LB2_OK;
    LB2_REQUIRE(h, out, "segment_dot null");
    cudaStream_t s = (cudaStream_t)stream;
    if (nrows == 0) {                    // no rows: every sum is empty (and the empty inputs may have no data pointer)
        if (cudaMemsetAsync(out, 0, (size_t)nseg * c * sizeof(float), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "segment_dot memset%s", "");
        return LB2_OK;
    }
    LB2_REQUIRE(h, a && offsets && scratch, "segment_dot null");
    float* partial = (float*)scratch;
    // 16-byte loads need every row, and so the row pitch and the bases, on a 16-byte boundary
    const bool vec = c % 4 == 0 && ((uintptr_t)a | (uintptr_t)b | (uintptr_t)out | (uintptr_t)scratch) % 16 == 0;
    if (vec) {
        if (b) launch<float4, true>(s, a, b, order, offsets, nseg, nrows, c / 4, partial, out);
        else launch<float4, false>(s, a, b, order, offsets, nseg, nrows, c / 4, partial, out);
    } else {
        if (b) launch<float, true>(s, a, b, order, offsets, nseg, nrows, c, partial, out);
        else launch<float, false>(s, a, b, order, offsets, nseg, nrows, c, partial, out);
    }
    LB2_POST_LAUNCH(h, "k_segment_dot_chunks");
    k_segment_dot_reduce<<<cdiv(nseg * c, 256), 256, 0, s>>>(offsets, nseg, c, partial, out);
    LB2_POST_LAUNCH(h, "k_segment_dot_reduce");
    return LB2_OK;
}
