// Synchronised batch norm: training-mode statistics over the rows of every rank, as exact integer sums (include/lidiff_b200.h states
// the element formulas and the error bound).  Every value is rounded once to a fixed-point grid set by a per-channel maximum that the
// ranks combine with MAX; the grid values are summed in 64-bit integer words that the ranks combine with SUM.  Integer sums do not
// depend on the order of their terms, so the results depend on the multiset of rows only: not on the row order, the launch shape or
// the split of rows across ranks.  Only integer atomics (shared, then one per block and word in global memory).
#include "common.cuh"

namespace sbn {

constexpr int THREADS = 256;
constexpr unsigned long long M32 = 0xffffffffull;

// A block is R rows x c channels (R = 256 / c, at least 1): thread t owns channel t % c for all its rows, so its per-channel
// parameters load once and a block's reads of R consecutive rows are contiguous.
__host__ __device__ inline int rows_per_block(int c) { return c >= THREADS ? 1 : THREADS / c; }

__device__ __forceinline__ int exp_of(double m) {          // m < 2^e (m = 0: e = 0)
    int e;
    frexp(m, &e);
    return e;
}

__device__ __forceinline__ double pow2(int k) { return ldexp(1.0, k); }

// RN64(W / n) for W = sum_k w[k] 2^(32 k), 0 <= w[k] < 2^63, 1 <= n < 2^32: three fraction digits below W's digits make the quotient
// at least 2^65 when W >= 1, a 32-bit-digit long division gives it exactly, and its top 64 bits with the rest ORed into bit 0 round
// once to 53 bits (bits 0..10 lie below the rounding position, so a tie is seen exactly when every lower bit is 0)
template <int K>
__device__ double div_rn(const unsigned long long (&w)[K], unsigned long long n) {
    constexpr int D = K + 5;
    unsigned dig[D];
    dig[0] = dig[1] = dig[2] = 0u;
    unsigned long long carry = 0;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const unsigned long long acc = carry + w[k];
        dig[3 + k] = (unsigned)(acc & M32);
        carry = acc >> 32;
    }
    dig[3 + K] = (unsigned)(carry & M32);
    dig[4 + K] = (unsigned)(carry >> 32);
    unsigned q[D];
    unsigned long long rem = 0;
#pragma unroll
    for (int i = D - 1; i >= 0; --i) {
        const unsigned long long cur = (rem << 32) | dig[i];
        q[i] = (unsigned)(cur / n);
        rem = cur % n;
    }
    int top = D - 1;
    while (top >= 0 && q[top] == 0u) --top;
    if (top < 0) return 0.0;
    const unsigned long long hi = ((unsigned long long)q[top] << 32) | (top >= 1 ? q[top - 1] : 0u);
    const unsigned lo = top >= 2 ? q[top - 2] : 0u;
    const int lz = __clzll(hi);                                      // 0..31: q[top] != 0
    unsigned long long m = lz ? (hi << lz) | (lo >> (32 - lz)) : hi;
    bool sticky = rem != 0 || (lz ? (lo & ((1u << (32 - lz)) - 1u)) != 0u : lo != 0u);
    for (int i = top - 3; i >= 0; --i) sticky |= q[i] != 0u;
    m |= (unsigned long long)sticky;
    return ldexp(__ull2double_rn(m), 32 * (top - 1) - lz - 96);
}

// RN64(S / n) for S = hi 2^32 + lo (the words of a signed sum)
__device__ double signed_div_rn(long long hi, long long lo, unsigned long long n) {
    const __int128 s = ((__int128)hi << 32) + (__int128)lo;
    const unsigned __int128 u = s < 0 ? (unsigned __int128)(-s) : (unsigned __int128)s;
    const unsigned long long w[3] = {(unsigned long long)(u & M32), (unsigned long long)((u >> 32) & M32), (unsigned long long)(u >> 64)};
    const double r = div_rn<3>(w, n);
    return s < 0 ? -r : r;
}

// RN64(S) for the same words (a sum, not a mean)
__device__ double signed_to_double(long long hi, long long lo) { return signed_div_rn(hi, lo, 1ull); }

__device__ __forceinline__ double nan64() { return __longlong_as_double(0x7ff8000000000000ll); }

// the global row count the words are exact for: 1 <= N < 2^31 (the ranks' counts are summed on the device, so a larger N is only
// seen here; its statistics are NaN rather than wrapped words)
__device__ __forceinline__ bool count_ok(long long n) { return n > 0 && n < (1ll << 31); }

// the signed fixed-point value q = RN(v 2^s) (|q| <= 2^62) into the words hi (q >> 32, arithmetic) and lo (q & 0xffffffff)
__device__ __forceinline__ void add_q(double v, double scale, long long& hi, unsigned long long& lo) {
    const long long q = llrint(__dmul_rn(v, scale));
    hi += q >> 32;
    lo += (unsigned long long)q & M32;
}

__device__ __forceinline__ float max_bits_to_float(long long w) { return __uint_as_float((unsigned)w); }

// ---- forward ---------------------------------------------------------------------------------------------------------------------
__global__ void k_max(const float* __restrict__ x, int64_t n, int c, unsigned long long* __restrict__ w) {
    extern __shared__ unsigned long long sh[];
    unsigned* smax = (unsigned*)sh;
    unsigned* sflag = smax + c;
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    for (int i = threadIdx.x; i < c; i += blockDim.x) smax[i] = sflag[i] = 0u;
    __syncthreads();
    unsigned m = 0u, flag = 0u;
    for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) {
        const float v = __ldg(x + r * c + j);
        if (isfinite(v)) m = max(m, __float_as_uint(fabsf(v)));              // non-negative floats order like their bits
        else flag = 1u;
    }
    atomicMax(smax + j, m);
    atomicOr(sflag + j, flag);
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        if (smax[i]) atomicMax(w + 2 * i, (unsigned long long)smax[i]);
        if (sflag[i]) atomicMax(w + 2 * i + 1, 1ull);
    }
}

__global__ void k_sum(const float* __restrict__ x, int64_t n, int c, const long long* __restrict__ maxw,
                      unsigned long long* __restrict__ w) {
    extern __shared__ unsigned long long sh[];
    unsigned long long* shi = sh;
    unsigned long long* slo = sh + c;
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    for (int i = threadIdx.x; i < c; i += blockDim.x) shi[i] = slo[i] = 0ull;
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(w + 2 * c, (unsigned long long)n);
    long long hi = 0;
    unsigned long long lo = 0;
    if (j < c && lane < R && maxw[2 * j + 1] == 0) {
        const double scale = pow2(62 - exp_of(max_bits_to_float(maxw[2 * j])));
        for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) add_q((double)__ldg(x + r * c + j), scale, hi, lo);
    }
    atomicAdd(shi + j, (unsigned long long)hi);                               // two's complement: the wrapped sum is the signed sum
    atomicAdd(slo + j, lo);
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        atomicAdd(w + 2 * i, shi[i]);
        atomicAdd(w + 2 * i + 1, slo[i]);
    }
}

__global__ void k_mean(int c, const long long* __restrict__ maxw, const long long* __restrict__ sumw, double* __restrict__ mean) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= c) return;
    const long long n = sumw[2 * c];
    if (maxw[2 * j + 1] != 0 || !count_ok(n)) { mean[j] = nan64(); return; }
    const int s = 62 - exp_of(max_bits_to_float(maxw[2 * j]));
    mean[j] = ldexp(signed_div_rn(sumw[2 * j], sumw[2 * j + 1], (unsigned long long)n), -s);
}

// t of the deviations' grid: B = RN64(max|x| + |mean|) < 2^e, t = 62 - e
__device__ __forceinline__ int dev_shift(long long maxbits, double mu) {
    return 62 - exp_of(__dadd_rn((double)max_bits_to_float(maxbits), fabs(mu)));
}

__global__ void k_sumsq(const float* __restrict__ x, int64_t n, int c, const long long* __restrict__ maxw,
                        const double* __restrict__ mean, unsigned long long* __restrict__ w) {
    extern __shared__ unsigned long long sh[];
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    for (int i = threadIdx.x; i < 4 * c; i += blockDim.x) sh[i] = 0ull;
    __syncthreads();
    unsigned long long l[4] = {0ull, 0ull, 0ull, 0ull};
    if (j < c && lane < R && maxw[2 * j + 1] == 0) {
        const double mu = mean[j];
        const double scale = pow2(dev_shift(maxw[2 * j], mu));
        for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) {
            const double d = __dsub_rn((double)__ldg(x + r * c + j), mu);
            const long long p = llrint(__dmul_rn(d, scale));
            const unsigned long long a = (unsigned long long)(p < 0 ? -p : p);
            const unsigned long long sq_lo = a * a, sq_hi = __umul64hi(a, a);      // p^2 < 2^125: four 32-bit limbs
            l[0] += sq_lo & M32;
            l[1] += sq_lo >> 32;
            l[2] += sq_hi & M32;
            l[3] += sq_hi >> 32;
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) atomicAdd(sh + 4 * j + k, l[k]);
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * c; i += blockDim.x) atomicAdd(w + i, sh[i]);
}

__global__ void k_var(int c, const long long* __restrict__ maxw, const long long* __restrict__ sumw, const double* __restrict__ mean,
                      const long long* __restrict__ sqw, double eps, double momentum, float* __restrict__ running_mean,
                      float* __restrict__ running_var, double* __restrict__ var, double* __restrict__ invstd) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= c) return;
    const long long n = sumw[2 * c];
    const double mu = mean[j];
    double v = nan64();
    if (maxw[2 * j + 1] == 0 && count_ok(n)) {
        const unsigned long long w[4] = {(unsigned long long)sqw[4 * j], (unsigned long long)sqw[4 * j + 1],
                                         (unsigned long long)sqw[4 * j + 2], (unsigned long long)sqw[4 * j + 3]};
        v = ldexp(div_rn<4>(w, (unsigned long long)n), -2 * dev_shift(maxw[2 * j], mu));
    }
    var[j] = v;
    invstd[j] = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(v, eps)));
    if (running_mean) {
        const double keep = __dsub_rn(1.0, momentum);
        running_mean[j] = __double2float_rn(__dadd_rn(__dmul_rn(keep, (double)running_mean[j]), __dmul_rn(momentum, mu)));
        // unbiased: RN64(RN64(var n) / (n - 1)); n = 1 gives 0 / 0 = NaN
        const double unbiased = __ddiv_rn(__dmul_rn(v, (double)n), (double)(n - 1));
        running_var[j] = __double2float_rn(__dadd_rn(__dmul_rn(keep, (double)running_var[j]), __dmul_rn(momentum, unbiased)));
    }
}

__global__ void k_apply(const float* __restrict__ x, int64_t n, int c, const double* __restrict__ mean, const double* __restrict__ invstd,
                        const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y) {
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    if (lane >= R) return;
    const double mu = mean[j], is = invstd[j];
    const double g = gamma ? (double)gamma[j] : 1.0, b = beta ? (double)beta[j] : 0.0;
    for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) {
        const double xh = __dmul_rn(__dsub_rn((double)__ldg(x + r * c + j), mu), is);
        y[r * c + j] = __double2float_rn(__dadd_rn(__dmul_rn(xh, g), b));
    }
}

// ---- backward --------------------------------------------------------------------------------------------------------------------
// g = RN64(dy xhat), xhat = RN64(RN64(x - mean) invstd) as in the forward
__device__ __forceinline__ double dy_xhat(float dy, float x, double mu, double is) {
    return __dmul_rn((double)dy, __dmul_rn(__dsub_rn((double)x, mu), is));
}

__global__ void k_bwd_max(const float* __restrict__ dy, const float* __restrict__ x, int64_t n, int c, const double* __restrict__ mean,
                          const double* __restrict__ invstd, unsigned long long* __restrict__ w) {
    extern __shared__ unsigned long long sh[];
    unsigned long long* sg = sh;
    unsigned* sdy = (unsigned*)(sh + c);
    unsigned* sflag = sdy + c;
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    for (int i = threadIdx.x; i < c; i += blockDim.x) { sg[i] = 0ull; sdy[i] = sflag[i] = 0u; }
    __syncthreads();
    unsigned mdy = 0u, flag = 0u;
    unsigned long long mg = 0ull;
    if (lane < R) {
        const double mu = mean[j], is = invstd[j];
        for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) {
            const float d = __ldg(dy + r * c + j);
            const double g = dy_xhat(d, __ldg(x + r * c + j), mu, is);
            if (isfinite(d) && isfinite(g)) {
                mdy = max(mdy, __float_as_uint(fabsf(d)));
                mg = max(mg, (unsigned long long)__double_as_longlong(fabs(g)));
            } else {
                flag = 1u;
            }
        }
    }
    atomicMax(sdy + j, mdy);
    atomicMax(sg + j, mg);
    atomicOr(sflag + j, flag);
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        if (sdy[i]) atomicMax(w + 3 * i, (unsigned long long)sdy[i]);
        if (sg[i]) atomicMax(w + 3 * i + 1, sg[i]);
        if (sflag[i]) atomicMax(w + 3 * i + 2, 1ull);
    }
}

__device__ __forceinline__ int dy_shift(long long w) { return 62 - exp_of(max_bits_to_float(w)); }
__device__ __forceinline__ int g_shift(long long w) { return 62 - exp_of(__longlong_as_double(w)); }

__global__ void k_bwd_sum(const float* __restrict__ dy, const float* __restrict__ x, int64_t n, int c, const double* __restrict__ mean,
                          const double* __restrict__ invstd, const long long* __restrict__ maxw, unsigned long long* __restrict__ w) {
    extern __shared__ unsigned long long sh[];
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    for (int i = threadIdx.x; i < 4 * c; i += blockDim.x) sh[i] = 0ull;
    __syncthreads();
    long long ahi = 0, bhi = 0;
    unsigned long long alo = 0, blo = 0;
    if (lane < R && maxw[3 * j + 2] == 0) {
        const double mu = mean[j], is = invstd[j];
        const double sa = pow2(dy_shift(maxw[3 * j])), sb = pow2(g_shift(maxw[3 * j + 1]));
        for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) {
            const float d = __ldg(dy + r * c + j);
            add_q((double)d, sa, ahi, alo);
            add_q(dy_xhat(d, __ldg(x + r * c + j), mu, is), sb, bhi, blo);
        }
    }
    atomicAdd(sh + 4 * j, (unsigned long long)ahi);
    atomicAdd(sh + 4 * j + 1, alo);
    atomicAdd(sh + 4 * j + 2, (unsigned long long)bhi);
    atomicAdd(sh + 4 * j + 3, blo);
    __syncthreads();
    for (int i = threadIdx.x; i < 4 * c; i += blockDim.x) atomicAdd(w + i, sh[i]);
}

// this rank's parameter gradients: dbeta = RN32(RN64(sum dy)), dgamma = RN32(RN64(sum dy xhat)) from the local words
__global__ void k_bwd_local(int c, const long long* __restrict__ maxw, const long long* __restrict__ w, float* __restrict__ dgamma,
                            float* __restrict__ dbeta) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= c) return;
    const bool bad = maxw[3 * j + 2] != 0;
    if (dbeta) dbeta[j] = bad ? (float)nan64() : __double2float_rn(ldexp(signed_to_double(w[4 * j], w[4 * j + 1]), -dy_shift(maxw[3 * j])));
    if (dgamma)
        dgamma[j] = bad ? (float)nan64() : __double2float_rn(ldexp(signed_to_double(w[4 * j + 2], w[4 * j + 3]), -g_shift(maxw[3 * j + 1])));
}

__global__ void k_bwd_apply(const float* __restrict__ dy, const float* __restrict__ x, int64_t n, int c, const double* __restrict__ mean,
                            const double* __restrict__ invstd, const float* __restrict__ gamma, const long long* __restrict__ maxw,
                            const long long* __restrict__ w, const long long* __restrict__ count, float* __restrict__ dx) {
    extern __shared__ unsigned long long sh[];
    double* smdy = (double*)sh;
    double* smg = smdy + c;
    const int R = rows_per_block(c), j = threadIdx.x % c, lane = threadIdx.x / c;
    const long long ntot = *count;
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        if (maxw[3 * i + 2] != 0 || !count_ok(ntot)) {
            smdy[i] = smg[i] = nan64();
        } else {
            smdy[i] = ldexp(signed_div_rn(w[4 * i], w[4 * i + 1], (unsigned long long)ntot), -dy_shift(maxw[3 * i]));
            smg[i] = ldexp(signed_div_rn(w[4 * i + 2], w[4 * i + 3], (unsigned long long)ntot), -g_shift(maxw[3 * i + 1]));
        }
    }
    __syncthreads();
    if (lane >= R) return;
    const double mu = mean[j], is = invstd[j], mdy = smdy[j], mg = smg[j];
    const double k = __dmul_rn(gamma ? (double)gamma[j] : 1.0, is);
    for (int64_t r = (int64_t)blockIdx.x * R + lane; r < n; r += (int64_t)gridDim.x * R) {
        const float d = __ldg(dy + r * c + j);
        const double xh = __dmul_rn(__dsub_rn((double)__ldg(x + r * c + j), mu), is);
        dx[r * c + j] = __double2float_rn(__dmul_rn(k, __dsub_rn(__dsub_rn((double)d, mdy), __dmul_rn(xh, mg))));
    }
}

struct Launch {
    int grid, block;
};

static Launch shape(const Lb2Handle* h, int64_t n, int c) {
    const int R = rows_per_block(c);
    const int64_t blocks = std::min<int64_t>(cdiv(n, R), (int64_t)h->num_sms * 8);
    return {(int)std::max<int64_t>(blocks, 1), R * c};
}

}  // namespace sbn

#define SBN_CHECK(h, n, c) \
    LB2_REQUIRE(h, h && (n) >= 0 && (n) < (1ll << 31) && (c) >= 1 && (c) <= 1024, "sync_bn: 0 <= n < 2^31, 1 <= c <= 1024")

extern "C" int lb2_sync_bn_max(void* handle, void* stream, const float* x, int64_t n, int32_t c, int64_t* max_words) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, max_words && (n == 0 || x), "sync_bn_max null");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(max_words, 0, 2 * (size_t)c * sizeof(int64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "sync_bn memset%s", "");
    if (n == 0) return LB2_OK;
    const Launch L = shape(h, n, c);
    k_max<<<L.grid, L.block, 2 * c * sizeof(unsigned), s>>>(x, n, c, (unsigned long long*)max_words);
    LB2_POST_LAUNCH(h, "k_sync_bn_max");
    return LB2_OK;
}

extern "C" int lb2_sync_bn_sum(void* handle, void* stream, const float* x, int64_t n, int32_t c, const int64_t* max_words,
                               int64_t* sum_words) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, max_words && sum_words && (n == 0 || x), "sync_bn_sum null");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(sum_words, 0, (2 * (size_t)c + 1) * sizeof(int64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "sync_bn memset%s", "");
    if (n == 0) return LB2_OK;
    const Launch L = shape(h, n, c);
    k_sum<<<L.grid, L.block, 2 * c * sizeof(unsigned long long), s>>>(x, n, c, (const long long*)max_words, (unsigned long long*)sum_words);
    LB2_POST_LAUNCH(h, "k_sync_bn_sum");
    return LB2_OK;
}

extern "C" int lb2_sync_bn_sumsq(void* handle, void* stream, const float* x, int64_t n, int32_t c, const int64_t* max_words,
                                 const int64_t* sum_words, double* mean, int64_t* sq_words) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, max_words && sum_words && mean && sq_words && (n == 0 || x), "sync_bn_sumsq null");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(sq_words, 0, 4 * (size_t)c * sizeof(int64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "sync_bn memset%s", "");
    k_mean<<<cdiv(c, 128), 128, 0, s>>>(c, (const long long*)max_words, (const long long*)sum_words, mean);
    LB2_POST_LAUNCH(h, "k_sync_bn_mean");
    if (n == 0) return LB2_OK;
    const Launch L = shape(h, n, c);
    k_sumsq<<<L.grid, L.block, 4 * c * sizeof(unsigned long long), s>>>(x, n, c, (const long long*)max_words, mean,
                                                                         (unsigned long long*)sq_words);
    LB2_POST_LAUNCH(h, "k_sync_bn_sumsq");
    return LB2_OK;
}

extern "C" int lb2_sync_bn_apply(void* handle, void* stream, const float* x, int64_t n, int32_t c, const int64_t* max_words,
                                 const int64_t* sum_words, const double* mean, const int64_t* sq_words, const float* gamma,
                                 const float* beta, double eps, double momentum, float* running_mean, float* running_var, double* var,
                                 double* invstd, float* y) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, max_words && sum_words && mean && sq_words && var && invstd && (n == 0 || (x && y)), "sync_bn_apply null");
    LB2_REQUIRE(h, (running_mean == nullptr) == (running_var == nullptr), "sync_bn_apply: both running statistics or neither");
    cudaStream_t s = (cudaStream_t)stream;
    k_var<<<cdiv(c, 128), 128, 0, s>>>(c, (const long long*)max_words, (const long long*)sum_words, mean, (const long long*)sq_words, eps,
                                       momentum, running_mean, running_var, var, invstd);
    LB2_POST_LAUNCH(h, "k_sync_bn_var");
    if (n == 0) return LB2_OK;
    const Launch L = shape(h, n, c);
    k_apply<<<L.grid, L.block, 0, s>>>(x, n, c, mean, invstd, gamma, beta, y);
    LB2_POST_LAUNCH(h, "k_sync_bn_apply");
    return LB2_OK;
}

extern "C" int lb2_sync_bn_backward_max(void* handle, void* stream, const float* dy, const float* x, int64_t n, int32_t c,
                                        const double* mean, const double* invstd, int64_t* max_words) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, mean && invstd && max_words && (n == 0 || (dy && x)), "sync_bn_backward_max null");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(max_words, 0, 3 * (size_t)c * sizeof(int64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "sync_bn memset%s", "");
    if (n == 0) return LB2_OK;
    const Launch L = shape(h, n, c);
    k_bwd_max<<<L.grid, L.block, c * (sizeof(unsigned long long) + 2 * sizeof(unsigned)), s>>>(dy, x, n, c, mean, invstd,
                                                                                                (unsigned long long*)max_words);
    LB2_POST_LAUNCH(h, "k_sync_bn_backward_max");
    return LB2_OK;
}

extern "C" int lb2_sync_bn_backward_sum(void* handle, void* stream, const float* dy, const float* x, int64_t n, int32_t c,
                                        const double* mean, const double* invstd, const int64_t* max_words, int64_t* sum_words,
                                        float* dgamma, float* dbeta) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, mean && invstd && max_words && sum_words && (n == 0 || (dy && x)), "sync_bn_backward_sum null");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(sum_words, 0, 4 * (size_t)c * sizeof(int64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "sync_bn memset%s", "");
    if (n > 0) {
        const Launch L = shape(h, n, c);
        k_bwd_sum<<<L.grid, L.block, 4 * c * sizeof(unsigned long long), s>>>(dy, x, n, c, mean, invstd, (const long long*)max_words,
                                                                               (unsigned long long*)sum_words);
        LB2_POST_LAUNCH(h, "k_sync_bn_backward_sum");
    }
    if (dgamma || dbeta) {
        k_bwd_local<<<cdiv(c, 128), 128, 0, s>>>(c, (const long long*)max_words, (const long long*)sum_words, dgamma, dbeta);
        LB2_POST_LAUNCH(h, "k_sync_bn_backward_local");
    }
    return LB2_OK;
}

extern "C" int lb2_sync_bn_backward_apply(void* handle, void* stream, const float* dy, const float* x, int64_t n, int32_t c,
                                          const double* mean, const double* invstd, const float* gamma, const int64_t* max_words,
                                          const int64_t* sum_words, const int64_t* count, float* dx) {
    using namespace sbn;
    Lb2Handle* h = (Lb2Handle*)handle;
    SBN_CHECK(h, n, c);
    LB2_REQUIRE(h, mean && invstd && max_words && sum_words && count, "sync_bn_backward_apply null");
    if (n == 0) return LB2_OK;
    LB2_REQUIRE(h, dy && x && dx, "sync_bn_backward_apply null");
    cudaStream_t s = (cudaStream_t)stream;
    const Launch L = shape(h, n, c);
    k_bwd_apply<<<L.grid, L.block, 2 * c * sizeof(double), s>>>(dy, x, n, c, mean, invstd, gamma, (const long long*)max_words,
                                                                (const long long*)sum_words, (const long long*)count, dx);
    LB2_POST_LAUNCH(h, "k_sync_bn_backward_apply");
    return LB2_OK;
}
