// Training / test samples of the diffusion network — stands behind lidiff/datasets/dataloader/SemanticKITTITemporal.py:82-105 (the
// scan's label / range / height filter, the map crop about the scan pose and its transform into the scan frame) and
// lidiff/utils/collations.py:44-51 (the 10 m viewpoint grid of the partial scan and the map points it includes), and the refinement
// network's samples (the end of this file).
// Every call is an order-preserving compaction: a count pass, a scan of the block totals, and an emit pass that evaluates the same
// inline predicate again and writes the kept rows at block offset + rank within the block.  Integer arithmetic decides every output
// position, so the output is deterministic and in input order.  Rows are addressed with 64-bit indices (inputs up to 2^31 - 1 rows).
#include "common.cuh"
#include <math.h>

#define SEL_THREADS 256
#define SEL_ITEMS   8
#define SEL_TILE    (SEL_THREADS * SEL_ITEMS)
#define SEL_WARPS   (SEL_THREADS / 32)
#define SCAN_THREADS 1024
#define VP_AXIS_BITS 21                      // viewpoint cell keys: 3 x 21 bit cell indices, each in [0, 2^21)

static size_t sel_align(size_t bytes) { return (bytes + 255) / 256 * 256; }
static int64_t sel_blocks(int64_t n) { return (n + SEL_TILE - 1) / SEL_TILE; }

// ---------------------------------------------------------------------------------------------------
// order-preserving compaction of rows [0, n) under a predicate `sel(i, w)` that also yields the fp64 output row w
// ---------------------------------------------------------------------------------------------------
template <class Sel>
__global__ void __launch_bounds__(SEL_THREADS) k_sel_count(Sel sel, int64_t n, long long* __restrict__ bcount) {
    __shared__ int warp_cnt[SEL_WARPS];
    int64_t base = (int64_t)blockIdx.x * SEL_TILE;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < SEL_ITEMS; ++j) {
        int64_t i = base + j * SEL_THREADS + threadIdx.x;
        double3 w;
        cnt += (i < n) && sel(i, w);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, d);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int k = 0; k < SEL_WARPS; ++k) t += warp_cnt[k];
        bcount[blockIdx.x] = t;
    }
}

// single block: exclusive scan of the nblk block totals in place; d_count[0] = the grand total
__global__ void __launch_bounds__(SCAN_THREADS) k_sel_scan(long long* __restrict__ b, int64_t nblk, int32_t* __restrict__ d_count) {
    __shared__ long long part[SCAN_THREADS];
    int64_t per = (nblk + SCAN_THREADS - 1) / SCAN_THREADS;
    int64_t lo = threadIdx.x * per, hi = min(lo + per, nblk);
    long long s = 0;
    for (int64_t k = lo; k < hi; ++k) s += b[k];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int d = 1; d < SCAN_THREADS; d <<= 1) {           // Hillis-Steele inclusive scan of the thread sums
        long long v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    long long run = part[threadIdx.x] - s;
    for (int64_t k = lo; k < hi; ++k) { long long v = b[k]; b[k] = run; run += v; }
    if (threadIdx.x == SCAN_THREADS - 1) d_count[0] = (int32_t)part[SCAN_THREADS - 1];
}

// item j of thread t is row base + j * SEL_THREADS + t: its rank in the block counts every kept row of the earlier stripes and the
// kept rows of stripe j held by lower threads
template <class Sel>
__global__ void __launch_bounds__(SEL_THREADS) k_sel_emit(Sel sel, int64_t n, const long long* __restrict__ boff, double* __restrict__ out) {
    __shared__ int cnt[SEL_ITEMS * SEL_WARPS];
    int64_t base = (int64_t)blockIdx.x * SEL_TILE;
    int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    unsigned lt = (1u << lane) - 1u;
    double3 w[SEL_ITEMS];
    bool f[SEL_ITEMS];
    int before[SEL_ITEMS];
#pragma unroll
    for (int j = 0; j < SEL_ITEMS; ++j) {
        int64_t i = base + j * SEL_THREADS + threadIdx.x;
        f[j] = (i < n) && sel(i, w[j]);
        unsigned bal = __ballot_sync(0xffffffffu, f[j]);
        before[j] = __popc(bal & lt);
        if (lane == 0) cnt[j * SEL_WARPS + wp] = __popc(bal);
    }
    __syncthreads();
    if (wp == 0) {                       // exclusive scan of the SEL_ITEMS x SEL_WARPS warp counts in (stripe, warp) order
        const int per = SEL_ITEMS * SEL_WARPS / 32;
        int v[per], t = 0;
#pragma unroll
        for (int k = 0; k < per; ++k) { v[k] = cnt[lane * per + k]; t += v[k]; }
        int incl = t;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
        int run = incl - t;
#pragma unroll
        for (int k = 0; k < per; ++k) { cnt[lane * per + k] = run; run += v[k]; }
    }
    __syncthreads();
    long long off = boff[blockIdx.x];
#pragma unroll
    for (int j = 0; j < SEL_ITEMS; ++j) {
        if (!f[j]) continue;
        long long r = off + cnt[j * SEL_WARPS + wp] + before[j];
        out[3 * r] = w[j].x; out[3 * r + 1] = w[j].y; out[3 * r + 2] = w[j].z;
    }
}

template <class Sel>
static int sel_compact(Lb2Handle* h, cudaStream_t s, const Sel& sel, int64_t n, long long* boff, double* out, int32_t* d_count) {
    if (n == 0) {
        if (cudaMemsetAsync(d_count, 0, sizeof(int32_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
        return LB2_OK;
    }
    int64_t nblk = sel_blocks(n);
    k_sel_count<<<(unsigned)nblk, SEL_THREADS, 0, s>>>(sel, n, boff);
    LB2_POST_LAUNCH(h, "k_sel_count");
    k_sel_scan<<<1, SCAN_THREADS, 0, s>>>(boff, nblk, d_count);
    LB2_POST_LAUNCH(h, "k_sel_scan");
    k_sel_emit<<<(unsigned)nblk, SEL_THREADS, 0, s>>>(sel, n, boff, out);
    LB2_POST_LAUNCH(h, "k_sel_emit");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// lb2_select_points
// ---------------------------------------------------------------------------------------------------
template <class T>
struct SelectPoints {
    const T* pts;
    const unsigned* labels;
    int stride;
    int range_mode;                 // LB2_RANGE_*
    float c32[3], rmin32, rmax32;
    double c64[3], rmin64, rmax64;
    int has_transform, has_z_min;
    double m[12], z_min;

    __device__ __forceinline__ bool operator()(int64_t i, double3& w) const {
        if (labels) {
            unsigned l = __ldg(labels + i) & 0xFFFFu;
            if (!(l > 1u && l < 252u)) return false;
        }
        const T* p = pts + i * stride;
        double x = (double)p[0], y = (double)p[1], z = (double)p[2];
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
        if (range_mode == LB2_RANGE_FP32) {
            float dx = __fsub_rn((float)x, c32[0]), dy = __fsub_rn((float)y, c32[1]), dz = __fsub_rn((float)z, c32[2]);
            float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            if (!(d > rmin32 && d < rmax32)) return false;
        } else if (range_mode == LB2_RANGE_FP64) {
            double dx = __dsub_rn(x, c64[0]), dy = __dsub_rn(y, c64[1]), dz = __dsub_rn(z, c64[2]);
            double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
            if (!(d > rmin64 && d < rmax64)) return false;
        }
        if (has_transform) {
            double c[3];
#pragma unroll
            for (int r = 0; r < 3; ++r)
                c[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4 * r], x), __dmul_rn(m[4 * r + 1], y)), __dmul_rn(m[4 * r + 2], z)),
                                 m[4 * r + 3]);
            x = c[0]; y = c[1]; z = c[2];
        }
        if (has_z_min && !(z > z_min)) return false;
        w = make_double3(x, y, z);
        return true;
    }
};

extern "C" size_t lb2_select_points_scratch_bytes(int64_t n) {
    return sel_align((size_t)(sel_blocks(n > 0 ? n : 1)) * sizeof(long long)) + 256;
}

template <class T>
static SelectPoints<T> make_select(const void* points, const uint32_t* labels, int32_t stride, const lb2_select_desc& d) {
    SelectPoints<T> s;
    s.pts = (const T*)points; s.labels = (const unsigned*)labels; s.stride = stride;
    s.range_mode = d.range_mode;
    for (int k = 0; k < 3; ++k) { s.c64[k] = d.center[k]; s.c32[k] = (float)d.center[k]; }
    s.rmin64 = d.r_min; s.rmax64 = d.r_max;
    s.rmin32 = (float)d.r_min; s.rmax32 = (float)d.r_max;          // round to nearest, as numpy compares a float32 array with a float
    s.has_transform = d.has_transform; s.has_z_min = d.has_z_min; s.z_min = d.z_min;
    for (int k = 0; k < 12; ++k) s.m[k] = d.transform[k];
    return s;
}

extern "C" int lb2_select_points(void* handle, void* stream, const void* points, int32_t fp64, int64_t n, int32_t stride,
                                 const uint32_t* labels, const lb2_select_desc* desc, double* out, int32_t* d_count, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, desc != nullptr && d_count != nullptr, "null desc / d_count");
    LB2_REQUIRE(h, n >= 0 && n <= (int64_t)INT32_MAX, "n out of range (0 .. 2^31 - 1 rows)");
    LB2_REQUIRE(h, stride == 3 || stride == 4, "stride must be 3 or 4");
    LB2_REQUIRE(h, desc->range_mode >= LB2_RANGE_NONE && desc->range_mode <= LB2_RANGE_FP64, "range_mode");
    LB2_REQUIRE(h, n == 0 || (points && out && scratch), "null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    long long* boff = (long long*)scratch;
    if (fp64) return sel_compact(h, s, make_select<double>(points, labels, stride, *desc), n, boff, out, d_count);
    return sel_compact(h, s, make_select<float>(points, labels, stride, *desc), n, boff, out, d_count);
}

// ---------------------------------------------------------------------------------------------------
// lb2_viewpoint_filter
// ---------------------------------------------------------------------------------------------------
struct VpScratch {
    double* origin;             // [3] min bound of p_part - voxel / 2
    unsigned long long* keys;   // [cap] occupied cells
    long long* boff;            // block offsets of the compaction
};

static int64_t vp_cap(int32_t n_part) { int64_t c = 16; while (c < 2 * (int64_t)(n_part > 0 ? n_part : 1)) c <<= 1; return c; }

extern "C" size_t lb2_viewpoint_filter_scratch_bytes(int32_t n_part, int64_t n_full) {
    return 256 + sel_align((size_t)vp_cap(n_part) * 8) + sel_align((size_t)sel_blocks(n_full > 0 ? n_full : 1) * sizeof(long long)) + 256;
}

static VpScratch vp_carve(void* scratch, int32_t n_part) {
    char* p = (char*)scratch;
    VpScratch v;
    v.origin = (double*)p;
    v.keys = (unsigned long long*)(p + 256);
    v.boff = (long long*)(p + 256 + sel_align((size_t)vp_cap(n_part) * 8));
    return v;
}

// cell key of p: floor((p - origin) / voxel) per axis in fp64 (the shim's VoxelGrid); false when a cell index is outside [0, 2^21)
__device__ __forceinline__ bool vp_key(double x, double y, double z, const double* __restrict__ o, double voxel, unsigned long long& key) {
    double c[3] = {x, y, z};
    key = 0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        double f = floor(__ddiv_rn(__dsub_rn(c[r], o[r]), voxel));
        if (!(f >= 0.0 && f < (double)(1 << VP_AXIS_BITS))) return false;      // NaN fails too
        key = (key << VP_AXIS_BITS) | (unsigned long long)f;
    }
    return true;
}

// single block: origin = per-axis minimum of p_part - voxel / 2 (fmin is exact, so the order of the reduction does not matter)
__global__ void __launch_bounds__(1024) k_vp_origin(const double* __restrict__ part, int n, double voxel, double* __restrict__ origin) {
    __shared__ double red[3][32];
    double m[3] = {INFINITY, INFINITY, INFINITY};
    for (int i = threadIdx.x; i < n; i += blockDim.x)
#pragma unroll
        for (int r = 0; r < 3; ++r) m[r] = fmin(m[r], part[3 * (int64_t)i + r]);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) m[r] = fmin(m[r], __shfl_down_sync(0xffffffffu, m[r], d));
        if ((threadIdx.x & 31) == 0) red[r][threadIdx.x >> 5] = m[r];
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double v = INFINITY;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) v = fmin(v, red[threadIdx.x][k]);
        origin[threadIdx.x] = __dsub_rn(v, 0.5 * voxel);
    }
}

__global__ void k_vp_insert(const double* __restrict__ part, int n, double voxel, const double* __restrict__ origin,
                            unsigned long long* keys, unsigned cap, int32_t* __restrict__ d_out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long key;
    if (!vp_key(part[3 * (int64_t)i], part[3 * (int64_t)i + 1], part[3 * (int64_t)i + 2], origin, voxel, key)) {
        atomicOr(d_out + 1, 1);
        return;
    }
    unsigned mask = cap - 1u, s = lb2_hash(key) & mask;
    while (true) {
        unsigned long long kk = keys[s];
        if (kk == LB2_KEY_EMPTY) {
            kk = atomicCAS(keys + s, (unsigned long long)LB2_KEY_EMPTY, key);
            if (kk == LB2_KEY_EMPTY) return;
        }
        if (kk == key) return;
        s = (s + 1) & mask;
    }
}

struct ViewpointSel {
    const double* full;
    const double* origin;
    const unsigned long long* keys;
    unsigned mask;
    double voxel;

    __device__ __forceinline__ bool operator()(int64_t i, double3& w) const {
        double x = full[3 * i], y = full[3 * i + 1], z = full[3 * i + 2];
        unsigned long long key;
        if (!vp_key(x, y, z, origin, voxel, key)) return false;
        unsigned s = lb2_hash(key) & mask;
        while (true) {
            unsigned long long kk = keys[s];
            if (kk == key) break;
            if (kk == LB2_KEY_EMPTY) return false;
            s = (s + 1) & mask;
        }
        w = make_double3(x, y, z);
        return true;
    }
};

extern "C" int lb2_viewpoint_filter(void* handle, void* stream, const double* part, int32_t n_part, const double* full, int64_t n_full,
                                    double voxel_size, double* out, int32_t* d_out, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, d_out != nullptr && scratch != nullptr, "null d_out / scratch");
    LB2_REQUIRE(h, n_part >= 0 && n_full >= 0 && n_full <= (int64_t)INT32_MAX, "n_part / n_full out of range");
    LB2_REQUIRE(h, voxel_size > 0.0, "voxel_size must be > 0");
    LB2_REQUIRE(h, (n_part == 0 || part) && (n_full == 0 || (full && out)), "null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(d_out, 0, 2 * sizeof(int32_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    if (n_part == 0 || n_full == 0) return LB2_OK;       // an empty grid includes nothing
    VpScratch v = vp_carve(scratch, n_part);
    int64_t cap = vp_cap(n_part);
    if (cudaMemsetAsync(v.keys, 0xFF, (size_t)cap * 8, s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    k_vp_origin<<<1, 1024, 0, s>>>(part, n_part, voxel_size, v.origin);
    LB2_POST_LAUNCH(h, "k_vp_origin");
    k_vp_insert<<<cdiv(n_part, 256), 256, 0, s>>>(part, n_part, voxel_size, v.origin, v.keys, (unsigned)cap, d_out);
    LB2_POST_LAUNCH(h, "k_vp_insert");
    ViewpointSel sel{full, v.origin, v.keys, (unsigned)cap - 1u, voxel_size};
    return sel_compact(h, s, sel, n_full, v.boff, out, d_out);
}

// ---------------------------------------------------------------------------------------------------
// refinement samples — lidiff/utils/pcd_preprocess.py:78-129 (aggregate_pcds) and SemanticKITTITemporalAggr.py:69-99 (__getitem__)
// ---------------------------------------------------------------------------------------------------
// single block: d_out[0] = kept rows of [0, row) = the block offset of row's tile + the kept rows of that tile before `row`
template <class Sel>
__global__ void __launch_bounds__(SEL_THREADS) k_sel_rank_at(Sel sel, int64_t row, const long long* __restrict__ boff,
                                                             int32_t* __restrict__ d_out) {
    __shared__ int warp_cnt[SEL_WARPS];
    int64_t base = row / SEL_TILE * SEL_TILE;
    int cnt = 0;
    for (int64_t i = base + threadIdx.x; i < row; i += SEL_THREADS) {
        double3 w;
        cnt += sel(i, w);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, d);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = boff[row / SEL_TILE];
        for (int k = 0; k < SEL_WARPS; ++k) t += warp_cnt[k];
        d_out[0] = (int32_t)t;
    }
}

// p' = ((m0 x + m1 y) + m2 z) + m3 per output axis in fp64, every operation rounded: numpy's
// np.sum(np.expand_dims(hpoints, 2) * pose.T, axis=1) adds the four products of a row in column order (w = 1, so m3 * w = m3)
__device__ __forceinline__ double3 rigid64(const double* __restrict__ m, double x, double y, double z) {
    double c[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        c[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[4 * r], x), __dmul_rn(m[4 * r + 1], y)), __dmul_rn(m[4 * r + 2], z)), m[4 * r + 3]);
    return make_double3(c[0], c[1], c[2]);
}

struct AggregateSel {
    const float4* pts;
    const unsigned* labels;
    const lb2_segment* seg;
    int nseg;
    double undo[12];

    __device__ __forceinline__ bool operator()(int64_t i, double3& w) const {
        unsigned l = __ldg(labels + i) & 0xFFFFu;
        if (!(l < 252u)) return false;
        float4 p = __ldg(pts + i);
        float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)), __fmul_rn(p.z, p.z)));
        if (!(d > 3.5f)) return false;                 // NaN fails, +-inf passes (numpy's comparison)
        int lo = 0, hi = nseg - 1;                     // the last segment whose start is <= i (empty segments share a start)
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (__ldg(&seg[mid].start) <= i) lo = mid; else hi = mid - 1;
        }
        double m[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) m[k] = __ldg(&seg[lo].m[k]);
        double3 a = rigid64(m, (double)p.x, (double)p.y, (double)p.z);
        w = rigid64(undo, a.x, a.y, a.z);
        return true;
    }
};

extern "C" size_t lb2_aggregate_window_scratch_bytes(int64_t n) { return lb2_select_points_scratch_bytes(n); }

extern "C" int lb2_aggregate_window(void* handle, void* stream, const float* points, const uint32_t* labels, int64_t n,
                                    const lb2_segment* segments, int32_t nseg, const double* undo, int64_t split, double* out,
                                    int32_t* d_out, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, d_out != nullptr && undo != nullptr, "null d_out / undo");
    LB2_REQUIRE(h, n >= 0 && n <= (int64_t)INT32_MAX, "n out of range (0 .. 2^31 - 1 rows)");
    LB2_REQUIRE(h, nseg >= 1 && segments != nullptr, "at least one segment");
    LB2_REQUIRE(h, split >= 0 && split <= n, "split out of range (0 .. n)");
    LB2_REQUIRE(h, n == 0 || (points && labels && out && scratch), "null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(d_out, 0, 2 * sizeof(int32_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    if (n == 0) return LB2_OK;
    AggregateSel sel;
    sel.pts = (const float4*)points; sel.labels = (const unsigned*)labels; sel.seg = segments; sel.nseg = nseg;
    for (int k = 0; k < 12; ++k) sel.undo[k] = undo[k];
    long long* boff = (long long*)scratch;
    int rc = sel_compact(h, s, sel, n, boff, out, d_out);
    if (rc != LB2_OK) return rc;
    if (split == n) {                                  // every kept row comes before the split
        if (cudaMemcpyAsync(d_out + 1, d_out, sizeof(int32_t), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
            return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemcpyAsync");
        return LB2_OK;
    }
    k_sel_rank_at<<<1, SEL_THREADS, 0, s>>>(sel, split, boff, d_out + 1);
    LB2_POST_LAUNCH(h, "k_sel_rank_at");
    return LB2_OK;
}

// p + clip(sigma r, -clip, clip) (pcd_transforms.py:35-40: the scale, then numpy's clip = minimum(maximum(v, -clip), clip), then the
// sum), kept where the fp64 distance sqrt((x^2 + y^2) + z^2) < r_max; NaN and inf rows fail the test
struct JitterSel {
    const double* p;
    const double* r;
    double sigma, clip, r_max;

    __device__ __forceinline__ bool operator()(int64_t i, double3& w) const {
        double c[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            double j = fmin(fmax(__dmul_rn(sigma, __ldg(r + 3 * i + k)), -clip), clip);
            c[k] = __dadd_rn(j, __ldg(p + 3 * i + k));
        }
        double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(c[0], c[0]), __dmul_rn(c[1], c[1])), __dmul_rn(c[2], c[2])));
        if (!(d < r_max)) return false;
        w = make_double3(c[0], c[1], c[2]);
        return true;
    }
};

extern "C" size_t lb2_jitter_filter_scratch_bytes(int64_t n) { return lb2_select_points_scratch_bytes(n); }

extern "C" int lb2_jitter_filter(void* handle, void* stream, const double* points, const double* randn, int64_t n, double sigma,
                                 double clip, double max_range, double* out, int32_t* d_count, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, d_count != nullptr, "null d_count");
    LB2_REQUIRE(h, n >= 0 && n <= (int64_t)INT32_MAX, "n out of range (0 .. 2^31 - 1 rows)");
    LB2_REQUIRE(h, clip > 0.0, "clip must be > 0");
    LB2_REQUIRE(h, n == 0 || (points && randn && out && scratch), "null buffer");
    JitterSel sel{points, randn, sigma, clip, max_range};
    return sel_compact(h, (cudaStream_t)stream, sel, n, (long long*)scratch, out, d_count);
}

// ---- first occurrence per voxel (ME.utils.sparse_quantize(p / voxel, return_index=True) on fp64 rows) ----
struct VoxelFirstScratch {
    unsigned long long* keys;   // [cap] voxel keys (lb2_map_key_push packing)
    unsigned long long* claim;  // [cap] lowest row index of the slot's voxel
    long long* boff;            // block offsets of the compaction
};

static int64_t vf_cap(int64_t n) { int64_t c = 16; while (c < 2 * n) c <<= 1; return c; }

extern "C" size_t lb2_voxel_first_f64_scratch_bytes(int64_t n) {
    return 2 * sel_align((size_t)vf_cap(n) * 8) + sel_align((size_t)sel_blocks(n > 0 ? n : 1) * sizeof(long long)) + 256;
}

static VoxelFirstScratch vf_carve(void* scratch, int64_t n) {
    char* p = (char*)scratch;
    size_t t = sel_align((size_t)vf_cap(n) * 8);
    return VoxelFirstScratch{(unsigned long long*)p, (unsigned long long*)(p + t), (long long*)(p + 2 * t)};
}

// key of a row with finite coordinates: floor(p / voxel) per axis, the true fp64 quotient; false when an index is outside the key range
__device__ __forceinline__ bool vf_key(double x, double y, double z, double voxel, unsigned long long& key) {
    double c[3] = {x, y, z};
    key = 0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        double f = floor(__ddiv_rn(c[r], voxel));
        if (!lb2_map_cell_ok(f)) return false;
        key = lb2_map_key_push(key, (int)f);
    }
    return true;
}

// Rows with a NaN or inf coordinate are left out of the table: the reference gives them voxels of their own (no finite row floors to
// them) and its distance test drops them afterwards, so leaving them out changes no output row.
__global__ void k_vf_insert(const double* __restrict__ p, int64_t n, double voxel, unsigned long long* keys, unsigned long long* claim,
                            unsigned mask, int32_t* __restrict__ d_out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    if (!(isfinite(x) && isfinite(y) && isfinite(z))) return;
    unsigned long long key;
    if (!vf_key(x, y, z, voxel, key)) {
        atomicOr(d_out + 1, 1);
        return;
    }
    atomicMin(claim + lb2_key_insert(keys, mask, key), (unsigned long long)i);
}

struct VoxelFirstSel {
    const double* p;
    const unsigned long long* keys;
    const unsigned long long* claim;
    unsigned mask;
    double voxel, r_max;

    __device__ __forceinline__ bool operator()(int64_t i, double3& w) const {
        double x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
        if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
        unsigned long long key;
        if (!vf_key(x, y, z, voxel, key)) return false;
        unsigned s = lb2_hash(key) & mask;
        while (keys[s] != key) s = (s + 1) & mask;        // inserted by k_vf_insert
        if (claim[s] != (unsigned long long)i) return false;
        double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
        if (!(d < r_max)) return false;
        w = make_double3(x, y, z);
        return true;
    }
};

extern "C" int lb2_voxel_first_f64(void* handle, void* stream, const double* points, int64_t n, double voxel_size, double max_range,
                                   double* out, int32_t* d_out, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, d_out != nullptr, "null d_out");
    LB2_REQUIRE(h, n >= 0 && n <= (int64_t)INT32_MAX, "n out of range (0 .. 2^31 - 1 rows)");
    LB2_REQUIRE(h, voxel_size > 0.0, "voxel_size must be > 0");
    LB2_REQUIRE(h, n == 0 || (points && out && scratch), "null buffer");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(d_out, 0, 2 * sizeof(int32_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    if (n == 0) return LB2_OK;
    VoxelFirstScratch v = vf_carve(scratch, n);
    int64_t cap = vf_cap(n);
    // keys EMPTY and claims "none" are both all-ones: one clear of the two adjacent arrays
    if (cudaMemsetAsync(v.keys, 0xFF, 2 * sel_align((size_t)cap * 8), s) != cudaSuccess)
        return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    unsigned mask = (unsigned)(cap - 1);
    k_vf_insert<<<cdiv(n, 256), 256, 0, s>>>(points, n, voxel_size, v.keys, v.claim, mask, d_out);
    LB2_POST_LAUNCH(h, "k_vf_insert");
    VoxelFirstSel sel{points, v.keys, v.claim, mask, voxel_size, max_range};
    return sel_compact(h, s, sel, n, v.boff, out, d_out);
}
