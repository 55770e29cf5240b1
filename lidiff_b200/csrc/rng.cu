// numpy's legacy randn and torch's CPU randperm drawn on the device, bit for bit (lidiff_b200/rng.py).
//   * lb2_mt19937_words: the MT19937 word stream of either generator.  One CTA holds the 624-word state in shared memory; a twist is
//     three dependent phases (i < 227 reads only the old state; 227 <= i < 454 and 454 <= i < 624 read words the phase before wrote),
//     so two state buffers and three barriers per twist.  Tempered words are stored coalesced.
//   * lb2_legacy_gauss: numpy's legacy_gauss (polar method) over those words.  Attempt k uses words 4k .. 4k+3; accept flags and a
//     scan of the block totals give every accepted attempt its output pair.  log(r2) is evaluated in double-double; where the exact
//     value lies more than `band` ulp from a rounding midpoint, glibc's log (error < 0.519 ulp) returns its correct rounding, which is
//     the double-double's leading word.  The rest are resolved on the host with libm's log, the function numpy calls.
//   * lb2_randperm: torch's forward Fisher-Yates shuffle (z_i = word_i % (n - i); swap(r[i], r[i + z_i])) by deterministic
//     reservations (Shun, Gu, Blelloch, Fineman, Gibbons, SODA 2015): each round every open iteration reserves positions i and
//     i + z_i with an atomicMin of its index; an iteration that holds both swaps and closes.  The result is the sequential one.
#include "common.cuh"
#include <cooperative_groups.h>
#include <math.h>
#include <vector>

#define MT_N 624
#define MT_M 397
#define MT_THREADS 256

__device__ __forceinline__ uint32_t mt_mix(uint32_t a, uint32_t b, uint32_t src) {
    uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return src ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    return y ^ (y >> 18);
}

// one twist of `a` into `b` (the sequential in-place twist, restated on two buffers)
__device__ __forceinline__ void mt_twist(const uint32_t* a, uint32_t* b) {
    int i = threadIdx.x;
    if (i < MT_N - MT_M) b[i] = mt_mix(a[i], a[i + 1], a[i + MT_M]);                      // 0 .. 226: old words only
    __syncthreads();
    i += MT_N - MT_M;
    if (i < 2 * (MT_N - MT_M)) b[i] = mt_mix(a[i], a[i + 1], b[i - (MT_N - MT_M)]);     // 227 .. 453: reads 0 .. 226
    __syncthreads();
    i += MT_N - MT_M;
    if (i < MT_N - 1) b[i] = mt_mix(a[i], a[i + 1], b[i - (MT_N - MT_M)]);              // 454 .. 622: reads 227 .. 395
    else if (i == MT_N - 1) b[i] = mt_mix(a[i], b[0], b[MT_M - 1]);                       // 623: wraps to the new word 0
    __syncthreads();
}

__global__ void __launch_bounds__(MT_THREADS) k_mt_words(uint32_t* __restrict__ state, int pos, int64_t n, uint32_t* __restrict__ out) {
    __shared__ uint32_t sm[2][MT_N];
    for (int i = threadIdx.x; i < MT_N; i += MT_THREADS) sm[0][i] = state[i];
    __syncthreads();
    int cur = 0;
    int64_t done = 0;
    while (done < n) {
        if (pos == MT_N) { mt_twist(sm[cur], sm[cur ^ 1]); cur ^= 1; pos = 0; }
        int take = (int)min((int64_t)(MT_N - pos), n - done);
        for (int i = threadIdx.x; i < take; i += MT_THREADS) out[done + i] = mt_temper(sm[cur][pos + i]);
        done += take;
        pos += take;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < MT_N; i += MT_THREADS) state[i] = sm[cur][i];
}

extern "C" int lb2_mt19937_words(void* handle, void* stream, uint32_t* state, int32_t pos, int64_t n, uint32_t* out, int32_t* pos_out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, state != nullptr && pos_out != nullptr, "null state / pos_out");
    LB2_REQUIRE(h, pos >= 0 && pos <= MT_N, "pos out of range (0 .. 624)");
    LB2_REQUIRE(h, n >= 0, "n < 0");
    LB2_REQUIRE(h, n == 0 || out != nullptr, "null out");
    *pos_out = pos;
    if (n == 0) return LB2_OK;
    int64_t first = MT_N - pos;
    *pos_out = n <= first ? (int32_t)(pos + n) : (int32_t)((n - first - 1) % MT_N + 1);
    k_mt_words<<<1, MT_THREADS, 0, (cudaStream_t)stream>>>(state, pos, n, out);
    LB2_POST_LAUNCH(h, "k_mt_words");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// legacy Gaussian
// ---------------------------------------------------------------------------------------------------
#define GS_THREADS 256
#define GS_ITEMS   4
#define GS_TILE    (GS_THREADS * GS_ITEMS)
#define GS_WARPS   (GS_THREADS / 32)
#define GS_SCAN_THREADS 1024

struct GaussDevInfo {
    long long total;        // accepted attempts among the words
    long long k_last;       // the attempt of the last output pair
    unsigned long long deferred;
    double trailing;        // f * x1 of the last pair when the pair count is odd (and its log was not deferred)
};

struct GaussDeferred {
    double r2, x1, x2;
    long long rank;
};

static size_t gs_align(size_t b) { return (b + 255) / 256 * 256; }

// attempt k: x = 2 legacy_double - 1 from words 4k, 4k+1 (x1) and 4k+2, 4k+3 (x2); every step is exact but r2
__device__ __forceinline__ bool gs_attempt(const uint4* __restrict__ w, int64_t k, double& x1, double& x2, double& r2) {
    uint4 v = __ldg(w + k);
    double d1 = (double)(((unsigned long long)(v.x >> 5) << 26) + (v.y >> 6)) * 0x1p-53;
    double d2 = (double)(((unsigned long long)(v.z >> 5) << 26) + (v.w >> 6)) * 0x1p-53;
    x1 = __dsub_rn(__dmul_rn(2.0, d1), 1.0);
    x2 = __dsub_rn(__dmul_rn(2.0, d2), 1.0);
    r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));
    return r2 < 1.0 && r2 != 0.0;
}

// ---- double-double arithmetic (error-free transforms, no contraction) ----
struct dd { double hi, lo; };
__device__ __forceinline__ dd dd_two_sum(double a, double b) {
    double s = __dadd_rn(a, b), bb = __dsub_rn(s, a);
    return dd{s, __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb))};
}
__device__ __forceinline__ dd dd_fast(double a, double b) {
    double s = __dadd_rn(a, b);
    return dd{s, __dsub_rn(b, __dsub_rn(s, a))};
}
__device__ __forceinline__ dd dd_add(dd a, dd b) {
    dd s = dd_two_sum(a.hi, b.hi), t = dd_two_sum(a.lo, b.lo);
    s = dd_fast(s.hi, __dadd_rn(s.lo, t.hi));
    return dd_fast(s.hi, __dadd_rn(s.lo, t.lo));
}
__device__ __forceinline__ dd dd_mul(dd a, dd b) {
    double p = __dmul_rn(a.hi, b.hi), e = __fma_rn(a.hi, b.hi, -p);
    e = __dadd_rn(e, __dadd_rn(__dmul_rn(a.hi, b.lo), __dmul_rn(a.lo, b.hi)));
    return dd_fast(p, e);
}
__device__ __forceinline__ dd dd_mul_d(dd a, double b) { return dd_mul(a, dd{b, 0.0}); }
__device__ __forceinline__ dd dd_div(dd a, dd b) {
    double q1 = __ddiv_rn(a.hi, b.hi);
    dd r = dd_add(a, dd_mul_d(b, -q1));
    double q2 = __ddiv_rn(r.hi, b.hi);
    r = dd_add(r, dd_mul_d(b, -q2));
    double q3 = __ddiv_rn(r.hi, b.hi);
    dd q = dd_fast(q1, q2);
    return dd_add(q, dd{q3, 0.0});
}
__device__ __forceinline__ dd dd_recip_odd(int d) {        // 1 / d to double-double (the residual by fma is exact)
    double hi = __drcp_rn((double)d);
    return dd{hi, __ddiv_rn(__fma_rn(-(double)d, hi, 1.0), (double)d)};
}

// log(r2), 0 < r2 < 1, with relative error below 2^-68: r2 = m 2^e with m in [sqrt(1/2), sqrt(2)), log m = 2 atanh(s),
// s = (m - 1) / (m + 1), |s| <= 0.1716; the series in t = s^2 <= 0.0295 to t^16 (truncation < 2^-80), terms from t^3 in fp64
// (their rounding is below 2^-71 of the sum)
__device__ __forceinline__ dd dd_log(double r2) {
    int e;
    double m = frexp(r2, &e);
    if (m < 0.70710678118654752440) { m = __dmul_rn(m, 2.0); --e; }
    dd num{__dsub_rn(m, 1.0), 0.0};                       // exact (Sterbenz)
    dd s = dd_div(num, dd_two_sum(m, 1.0));
    dd t = dd_mul(s, s);
    double q = 1.0 / 33.0;
#pragma unroll
    for (int k = 15; k >= 3; --k) q = __dadd_rn(__dmul_rn(q, t.hi), 1.0 / (2 * k + 1));
    dd p = dd_add(dd_mul_d(t, q), dd_recip_odd(5));       // 1/5 + t q
    p = dd_add(dd_mul(p, t), dd_recip_odd(3));
    p = dd_add(dd_mul(p, t), dd{1.0, 0.0});
    dd lm = dd_mul(s, p);
    lm.hi = __dmul_rn(lm.hi, 2.0); lm.lo = __dmul_rn(lm.lo, 2.0);
    dd el = dd_mul(dd{(double)e, 0.0}, dd{0x1.62e42fefa39efp-1, 0x1.abc9e3b39803fp-56});
    return dd_add(el, lm);
}

// the correctly rounded log(r2), or false when the exact value may lie within band ulp of a rounding midpoint (or the result is a
// power of two, where the ulp changes)
__device__ __forceinline__ bool gs_log(double r2, double band, double& L) {
    dd v = dd_log(r2);
    double a = fabs(v.hi);
    long long bits = __double_as_longlong(a);
    if ((bits & 0xFFFFFFFFFFFFFll) == 0) return false;
    double ulp = __dsub_rn(__longlong_as_double(bits + 1), a);
    double dist = __dsub_rn(__dmul_rn(0.5, ulp), fabs(v.lo));
    L = v.hi;
    return dist > __dmul_rn(band, ulp);
}

__device__ __forceinline__ void gs_write(double* __restrict__ out, int64_t n_out, int hg, long long rank, double L, double r2, double x1,
                                         double x2, GaussDevInfo* info) {
    double f = __dsqrt_rn(__ddiv_rn(__dmul_rn(-2.0, L), r2));
    int64_t o = hg + 2 * rank;
    out[o] = __dmul_rn(f, x2);
    if (o + 1 < n_out) out[o + 1] = __dmul_rn(f, x1);
    else info->trailing = __dmul_rn(f, x1);
}

__global__ void __launch_bounds__(GS_THREADS) k_gauss_count(const uint4* __restrict__ w, int64_t n_att, long long* __restrict__ bcount) {
    __shared__ int warp_cnt[GS_WARPS];
    int64_t base = (int64_t)blockIdx.x * GS_TILE;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < GS_ITEMS; ++j) {
        int64_t k = base + j * GS_THREADS + threadIdx.x;
        double x1, x2, r2;
        cnt += (k < n_att) && gs_attempt(w, k, x1, x2, r2);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, d);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int k = 0; k < GS_WARPS; ++k) t += warp_cnt[k];
        bcount[blockIdx.x] = t;
    }
}

// single block: exclusive scan of the block totals in place; *total = the grand total
__global__ void __launch_bounds__(GS_SCAN_THREADS) k_gauss_scan(long long* __restrict__ b, int64_t nblk, long long* __restrict__ total) {
    __shared__ long long part[GS_SCAN_THREADS];
    int64_t per = (nblk + GS_SCAN_THREADS - 1) / GS_SCAN_THREADS;
    int64_t lo = threadIdx.x * per, hi = min(lo + per, nblk);
    long long s = 0;
    for (int64_t k = lo; k < hi; ++k) s += b[k];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = 1; d < GS_SCAN_THREADS; d <<= 1) {
        long long v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    long long run = part[threadIdx.x] - s;
    for (int64_t k = lo; k < hi; ++k) { long long v = b[k]; b[k] = run; run += v; }
    if (threadIdx.x == GS_SCAN_THREADS - 1) *total = part[GS_SCAN_THREADS - 1];
}

// accepted attempt of rank r < pairs: output pair r, or a deferred record when its log is within the band
__global__ void __launch_bounds__(GS_THREADS) k_gauss_emit(const uint4* __restrict__ w, int64_t n_att, const long long* __restrict__ boff,
                                                           long long pairs, double* __restrict__ out, int64_t n_out, int hg, double band,
                                                           GaussDevInfo* info, GaussDeferred* __restrict__ rec) {
    __shared__ int cnt[GS_ITEMS * GS_WARPS];
    long long off = boff[blockIdx.x];
    if (off >= pairs) return;                                       // uniform per block
    int64_t base = (int64_t)blockIdx.x * GS_TILE;
    int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    unsigned lt = (1u << lane) - 1u;
    bool f[GS_ITEMS];
    int before[GS_ITEMS];
#pragma unroll
    for (int j = 0; j < GS_ITEMS; ++j) {
        int64_t k = base + j * GS_THREADS + threadIdx.x;
        double x1, x2, r2;
        f[j] = (k < n_att) && gs_attempt(w, k, x1, x2, r2);
        unsigned bal = __ballot_sync(0xffffffffu, f[j]);
        before[j] = __popc(bal & lt);
        if (lane == 0) cnt[j * GS_WARPS + wp] = __popc(bal);
    }
    __syncthreads();
    if (wp == 0) {                       // exclusive scan of the GS_ITEMS x GS_WARPS warp counts in (stripe, warp) order
        int v = cnt[lane], incl = v;     // GS_ITEMS * GS_WARPS == 32
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
        cnt[lane] = incl - v;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < GS_ITEMS; ++j) {
        if (!f[j]) continue;
        long long r = off + cnt[j * GS_WARPS + wp] + before[j];
        if (r >= pairs) continue;
        int64_t k = base + j * GS_THREADS + threadIdx.x;
        if (r == pairs - 1) info->k_last = k;
        double x1, x2, r2, L;
        gs_attempt(w, k, x1, x2, r2);
        if (gs_log(r2, band, L)) {
            gs_write(out, n_out, hg, r, L, r2, x1, x2, info);
        } else {
            unsigned long long d = atomicAdd(&info->deferred, 1ull);
            rec[d] = GaussDeferred{r2, x1, x2, r};
        }
    }
}

__global__ void k_gauss_deferred(const GaussDeferred* __restrict__ rec, const double* __restrict__ logs, long long nd, double* __restrict__ out,
                                 int64_t n_out, int hg, GaussDevInfo* info) {
    long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= nd) return;
    GaussDeferred g = rec[d];
    gs_write(out, n_out, hg, g.rank, logs[d], g.r2, g.x1, g.x2, info);
}

__global__ void k_gauss_cached(double* out, double g) { out[0] = g; }

static int64_t gs_pairs(int64_t n_out, int hg) { return (n_out - hg + 1) / 2; }

extern "C" size_t lb2_legacy_gauss_scratch_bytes(int64_t n_words, int64_t n_out) {
    int64_t nblk = (n_words / 4 + GS_TILE - 1) / GS_TILE;
    int64_t pairs = n_out > 0 ? gs_pairs(n_out, 0) : 0;
    return gs_align(sizeof(GaussDevInfo)) + gs_align((size_t)(nblk > 0 ? nblk : 1) * 8) + gs_align((size_t)pairs * sizeof(GaussDeferred))
         + gs_align((size_t)pairs * 8);
}

extern "C" int lb2_legacy_gauss(void* handle, void* stream, const uint32_t* words, int64_t n_words, int64_t n_out, int32_t has_gauss,
                                double gauss, double band, double* out, Lb2GaussInfo* info, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, info != nullptr, "null info");
    LB2_REQUIRE(h, n_words >= 0 && n_out >= 0, "negative size");
    LB2_REQUIRE(h, band >= 0.0 && band <= 0.5, "band out of range (0 .. 0.5 ulp)");
    LB2_REQUIRE(h, n_out == 0 || (out && scratch), "null buffer");
    LB2_REQUIRE(h, n_words == 0 || (words && ((uintptr_t)words & 15) == 0), "words must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    int hg = has_gauss ? 1 : 0;
    *info = Lb2GaussInfo{0, 0, 0, hg, gauss};
    if (n_out == 0) return LB2_OK;
    if (hg) {
        k_gauss_cached<<<1, 1, 0, s>>>(out, gauss);
        LB2_POST_LAUNCH(h, "k_gauss_cached");
    }
    int64_t pairs = gs_pairs(n_out, hg);
    bool odd = ((n_out - hg) & 1) != 0;
    if (pairs == 0) {                                    // the cached value alone: numpy clears the cache
        info->has_gauss = 0; info->gauss = 0.0;
        return LB2_OK;
    }
    int64_t n_att = n_words / 4;
    if (n_att < pairs) { info->short_words = 1; return LB2_OK; }
    int64_t nblk = (n_att + GS_TILE - 1) / GS_TILE;
    char* p = (char*)scratch;
    GaussDevInfo* dinfo = (GaussDevInfo*)p;            p += gs_align(sizeof(GaussDevInfo));
    long long* boff = (long long*)p;                   p += gs_align((size_t)nblk * 8);
    GaussDeferred* rec = (GaussDeferred*)p;            p += gs_align((size_t)gs_pairs(n_out, 0) * sizeof(GaussDeferred));
    double* d_logs = (double*)p;
    if (cudaMemsetAsync(dinfo, 0, sizeof(GaussDevInfo), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    const uint4* w = (const uint4*)words;
    k_gauss_count<<<(unsigned)nblk, GS_THREADS, 0, s>>>(w, n_att, boff);
    LB2_POST_LAUNCH(h, "k_gauss_count");
    k_gauss_scan<<<1, GS_SCAN_THREADS, 0, s>>>(boff, nblk, &dinfo->total);
    LB2_POST_LAUNCH(h, "k_gauss_scan");
    k_gauss_emit<<<(unsigned)nblk, GS_THREADS, 0, s>>>(w, n_att, boff, pairs, out, n_out, hg, band, dinfo, rec);
    LB2_POST_LAUNCH(h, "k_gauss_emit");
    GaussDevInfo hi;                                     // host read 1: the attempts reached and the deferred count
    if (cudaMemcpyAsync(&hi, dinfo, sizeof(hi), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess)
        return lb2_fail(h, LB2_ERR_CUDA, "%s", "reading the attempt count");
    if (hi.total < pairs) { info->short_words = 1; return LB2_OK; }
    double trailing = hi.trailing;
    long long nd = (long long)hi.deferred;
    if (nd > 0) {                                        // host read 2: the deferred attempts, resolved with libm's log
        std::vector<GaussDeferred> hrec((size_t)nd);
        std::vector<double> logs((size_t)nd);
        if (cudaMemcpyAsync(hrec.data(), rec, (size_t)nd * sizeof(GaussDeferred), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
            cudaStreamSynchronize(s) != cudaSuccess)
            return lb2_fail(h, LB2_ERR_CUDA, "%s", "reading the deferred attempts");
        for (long long d = 0; d < nd; ++d) {
            volatile double L = log(hrec[d].r2);         // the libm call numpy's legacy_gauss makes
            logs[d] = L;
            if (odd && hrec[d].rank == pairs - 1) {
                volatile double t = -2.0 * L;
                volatile double q = t / hrec[d].r2;
                volatile double f = sqrt(q);
                trailing = f * hrec[d].x1;
            }
        }
        if (cudaMemcpyAsync(d_logs, logs.data(), (size_t)nd * 8, cudaMemcpyHostToDevice, s) != cudaSuccess)
            return lb2_fail(h, LB2_ERR_CUDA, "%s", "uploading the deferred logs");
        k_gauss_deferred<<<cdiv(nd, 256), 256, 0, s>>>(rec, d_logs, nd, out, n_out, hg, dinfo);
        LB2_POST_LAUNCH(h, "k_gauss_deferred");
        if (cudaStreamSynchronize(s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "k_gauss_deferred");
    }
    info->words_used = 4 * (hi.k_last + 1);
    info->deferred = nd;
    info->has_gauss = odd ? 1 : 0;
    info->gauss = odd ? trailing : 0.0;
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// randperm by deterministic reservations
// ---------------------------------------------------------------------------------------------------
#define RP_THREADS 256

// reservation of iteration i in round r: later rounds have smaller keys, so a stale reservation never wins and none is cleared
__device__ __forceinline__ unsigned long long rp_key(int r, int64_t i) {
    return ((unsigned long long)(0xFFFFFFFFu - (unsigned)r) << 32) | (unsigned long long)i;
}

__global__ void __launch_bounds__(RP_THREADS) k_randperm(const uint32_t* __restrict__ words, int64_t n, long long* __restrict__ out,
                                                         unsigned long long* __restrict__ res, int32_t* __restrict__ list0,
                                                         int32_t* __restrict__ list1, int32_t* __restrict__ cnt, int32_t* __restrict__ d_rounds) {
    namespace cg = cooperative_groups;
    cg::grid_group g = cg::this_grid();
    int64_t stride = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t i = t0; i < n; i += stride) {
        out[i] = i;
        res[i] = ~0ull;
        if (i < n - 1) list0[i] = (int32_t)i;
    }
    if (t0 == 0) { cnt[0] = 0; cnt[1] = 0; }
    g.sync();
    int64_t open = n - 1;
    int32_t *cur = list0, *nxt = list1;
    int r = 0;
    while (open > 0) {
        for (int64_t k = t0; k < open; k += stride) {
            int64_t i = cur[k], j = i + (int64_t)(__ldg(words + i) % (uint32_t)(n - i));
            unsigned long long key = rp_key(r, i);
            atomicMin(res + i, key);
            if (j != i) atomicMin(res + j, key);
        }
        g.sync();
        for (int64_t k = t0; k < open; k += stride) {
            int64_t i = cur[k], j = i + (int64_t)(__ldg(words + i) % (uint32_t)(n - i));
            unsigned long long key = rp_key(r, i);
            if (res[i] == key && res[j] == key) {
                long long a = out[i];
                out[i] = out[j];
                out[j] = a;
            } else {
                nxt[atomicAdd(cnt + (r & 1), 1)] = (int32_t)i;
            }
        }
        g.sync();
        open = *(volatile int32_t*)(cnt + (r & 1));
        if (t0 == 0) cnt[(r + 1) & 1] = 0;            // read by every thread before this round's first barrier
        int32_t* tmp = cur; cur = nxt; nxt = tmp;
        ++r;
    }
    if (t0 == 0 && d_rounds) *d_rounds = r;
}

static size_t rp_res_bytes(int64_t n) { return gs_align((size_t)n * 8); }
static size_t rp_list_bytes(int64_t n) { return gs_align((size_t)n * 4); }

extern "C" size_t lb2_randperm_scratch_bytes(int64_t n) {
    if (n < 0) n = 0;
    return rp_res_bytes(n) + 2 * rp_list_bytes(n) + 256;
}

extern "C" int lb2_randperm(void* handle, void* stream, const uint32_t* words, int64_t n, int64_t* out, int32_t* d_rounds, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, n >= 0, "n < 0");
    LB2_REQUIRE(h, n < LB2_RANDPERM_MAX_N, "n >= 2^32 / 20: torch draws 64-bit words there");
    LB2_REQUIRE(h, n == 0 || out != nullptr, "null out");
    LB2_REQUIRE(h, n < 2 || (words && scratch), "null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    if (n < 2) {
        if (d_rounds && cudaMemsetAsync(d_rounds, 0, sizeof(int32_t), s) != cudaSuccess)
            return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
        if (n == 1 && cudaMemsetAsync(out, 0, sizeof(int64_t), s) != cudaSuccess)
            return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
        return LB2_OK;
    }
    char* p = (char*)scratch;
    unsigned long long* res = (unsigned long long*)p;  p += rp_res_bytes(n);
    int32_t* list0 = (int32_t*)p;                     p += rp_list_bytes(n);
    int32_t* list1 = (int32_t*)p;                     p += rp_list_bytes(n);
    int32_t* cnt = (int32_t*)p;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_randperm, RP_THREADS, 0) != cudaSuccess || per_sm < 1)
        return lb2_fail(h, LB2_ERR_CUDA, "%s", "k_randperm occupancy");
    int64_t want = (n + RP_THREADS - 1) / RP_THREADS;
    unsigned grid = (unsigned)min((int64_t)per_sm * h->num_sms, want);
    long long* o = (long long*)out;
    void* args[] = {(void*)&words, (void*)&n, (void*)&o, (void*)&res, (void*)&list0, (void*)&list1, (void*)&cnt, (void*)&d_rounds};
    cudaError_t e = cudaLaunchCooperativeKernel((const void*)k_randperm, dim3(grid), dim3(RP_THREADS), args, 0, s);
    h->launches++;
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s: %s", "k_randperm (cooperative launch)", cudaGetErrorString(e));
    return LB2_OK;
}
