// SemanticKITTI scene-completion voxel grids (lidiff_b200/ssc.py): grids -> voxel centres, points -> packed grids, and the
// benchmark's completion counts, in the format include/lidiff_b200.h pins.  Integer and bit work over 2^21 voxels per grid.
//   * k_ssc_count_{labels,bits}: one 32-voxel word per warp (labels: one voxel per lane and a ballot) or per thread (bits: the
//     word's bytes are MSB first, so a per-byte bit reversal gives the voxels in ascending order); writes the occupancy mask in
//     ascending voxel order and its popcount.
//   * k_ssc_scan: one block per grid, an exclusive scan of the 65 536 word counts in place; k_ssc_offsets chains the grids' totals.
//   * k_ssc_emit: one thread per voxel; a point's row is its grid's offset + its word's offset + the set bits below it, so the
//     output needs no atomics and comes out in ascending voxel order.
//   * k_ssc_voxelize: one thread per point, atomicOr into the packed grid, dropped rows counted once per warp and grid.
//   * k_ssc_confusion: one word per warp iteration, popcounts of TP / FP / FN, one integer atomic per warp and count at the end.
#include "common.cuh"

#define SSC_SCAN_THREADS 1024
#define SSC_SCAN_PER_THREAD (LB2_SSC_WORDS / SSC_SCAN_THREADS)     // 64

static_assert(LB2_SSC_VOXELS == LB2_SSC_DIM_X * LB2_SSC_DIM_Y * LB2_SSC_DIM_Z, "grid size");
static_assert(LB2_SSC_WORDS * 32 == LB2_SSC_VOXELS, "word count");

// bit (v & 31) ^ 7 of a device word holds voxel v (MSB-first bytes); this returns the word with voxel 32 w + k at bit k
__device__ __forceinline__ unsigned ssc_ascending(unsigned word) { return __byte_perm(__brev(word), 0, 0x0123); }

__device__ __forceinline__ bool ssc_occupied(unsigned label) { return label != 0 && label != LB2_SSC_IGNORE; }

__global__ void __launch_bounds__(256) k_ssc_count_labels(const uint16_t* __restrict__ labels, unsigned* __restrict__ masks,
                                                          unsigned* __restrict__ counts) {
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // a grid's voxels are a multiple of the block
    const unsigned m = __ballot_sync(0xffffffffu, ssc_occupied(__ldg(labels + v)));
    if ((threadIdx.x & 31) == 0) {
        masks[v >> 5] = m;
        counts[v >> 5] = __popc(m);
    }
}

__global__ void __launch_bounds__(256) k_ssc_count_bits(const unsigned* __restrict__ bits, long long n_words, unsigned* __restrict__ masks,
                                                        unsigned* __restrict__ counts) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    const unsigned m = ssc_ascending(__ldg(bits + w));
    masks[w] = m;
    counts[w] = __popc(m);
}

// counts of grid blockIdx.x -> their exclusive prefix sums in place; total[g] = the grid's occupied voxels
__global__ void __launch_bounds__(SSC_SCAN_THREADS) k_ssc_scan(unsigned* __restrict__ counts, long long* __restrict__ total) {
    __shared__ unsigned warp_sum[32];
    uint4* c = (uint4*)(counts + (long long)blockIdx.x * LB2_SSC_WORDS + threadIdx.x * SSC_SCAN_PER_THREAD);
    unsigned s = 0;
#pragma unroll 4
    for (int q = 0; q < SSC_SCAN_PER_THREAD / 4; ++q) {
        const uint4 x = c[q];
        s += x.x + x.y + x.z + x.w;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        unsigned t = warp_sum[lane], ti = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, ti, o);
            if (lane >= o) ti += y;
        }
        warp_sum[lane] = ti - t;                                     // exclusive prefix of the warps
        if (lane == 31) total[blockIdx.x] = ti;
    }
    __syncthreads();
    unsigned run = warp_sum[warp] + inc - s;
#pragma unroll 4
    for (int q = 0; q < SSC_SCAN_PER_THREAD / 4; ++q) {
        const uint4 x = c[q];
        uint4 y;
        y.x = run; run += x.x;
        y.y = run; run += x.y;
        y.z = run; run += x.z;
        y.w = run; run += x.w;
        c[q] = y;
    }
}

__global__ void k_ssc_offsets(const long long* __restrict__ total, long long n_grids, long long* __restrict__ offsets) {
    long long o = 0;
    offsets[0] = 0;
    for (long long g = 0; g < n_grids; ++g) {
        o += total[g];
        offsets[g + 1] = o;
    }
}

__device__ __forceinline__ double ssc_centre(int idx, double lo) {
    return __dadd_rn(lo, __dmul_rn(__dadd_rn((double)idx, 0.5), LB2_SSC_VOXEL));
}

__global__ void __launch_bounds__(256) k_ssc_emit(const unsigned* __restrict__ masks, const unsigned* __restrict__ word_off,
                                                  const long long* __restrict__ offsets, double* __restrict__ out) {
    const long long gv = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // the grid's voxel count is a multiple of the block
    const unsigned m = __ldg(masks + (gv >> 5));
    const int lane = (int)(gv & 31);
    if (!((m >> lane) & 1u)) return;
    const long long g = gv / LB2_SSC_VOXELS;
    const int u = (int)(gv - g * LB2_SSC_VOXELS);
    const long long row = __ldg(offsets + g) + __ldg(word_off + (gv >> 5)) + __popc(m & ((1u << lane) - 1u));
    const int i = u / (LB2_SSC_DIM_Y * LB2_SSC_DIM_Z), j = (u / LB2_SSC_DIM_Z) % LB2_SSC_DIM_Y, k = u % LB2_SSC_DIM_Z;
    out[3 * row] = ssc_centre(i, LB2_SSC_MIN_X);
    out[3 * row + 1] = ssc_centre(j, LB2_SSC_MIN_Y);
    out[3 * row + 2] = ssc_centre(k, LB2_SSC_MIN_Z);
}

// floor((p - lo) / 0.2), as a double so that any finite p compares correctly against the extent
__device__ __forceinline__ double ssc_index(double p, double lo) { return floor(__ddiv_rn(__dsub_rn(p, lo), LB2_SSC_VOXEL)); }

__global__ void __launch_bounds__(256) k_ssc_voxelize(const double* __restrict__ pts, const long long* __restrict__ offsets, long long n_grids,
                                                      long long n, unsigned* __restrict__ bits, lb2_ssc_voxel_info* __restrict__ info) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long g = -1;
    bool non_finite = false, outside = false;
    if (i < n) {
        long long lo = 0, hi = n_grids - 1;                              // the last g with offsets[g] <= i
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if (__ldg(offsets + mid) <= i) lo = mid; else hi = mid - 1;
        }
        g = lo;
        const double x = __ldg(pts + 3 * i), y = __ldg(pts + 3 * i + 1), z = __ldg(pts + 3 * i + 2);
        non_finite = !(isfinite(x) && isfinite(y) && isfinite(z));
        if (!non_finite) {
            const double fx = ssc_index(x, LB2_SSC_MIN_X), fy = ssc_index(y, LB2_SSC_MIN_Y), fz = ssc_index(z, LB2_SSC_MIN_Z);
            outside = !(fx >= 0.0 && fx < LB2_SSC_DIM_X && fy >= 0.0 && fy < LB2_SSC_DIM_Y && fz >= 0.0 && fz < LB2_SSC_DIM_Z);
            if (!outside) {
                const int v = ((int)fx * LB2_SSC_DIM_Y + (int)fy) * LB2_SSC_DIM_Z + (int)fz;
                atomicOr(bits + g * LB2_SSC_WORDS + (v >> 5), 1u << ((v & 31) ^ 7));
            }
        }
    }
    const unsigned same = __match_any_sync(0xffffffffu, g);
    const unsigned nf = __ballot_sync(0xffffffffu, non_finite) & same, out = __ballot_sync(0xffffffffu, outside) & same;
    if (g >= 0 && (int)(threadIdx.x & 31) == __ffs(same) - 1) {
        if (nf) atomicAdd((unsigned long long*)&info[g].non_finite, (unsigned long long)__popc(nf));
        if (out) atomicAdd((unsigned long long*)&info[g].outside, (unsigned long long)__popc(out));
    }
}

#define SSC_CONF_BLOCKS 64         // blocks per grid: 512 warps, 128 words each

__global__ void __launch_bounds__(256) k_ssc_confusion(const unsigned* __restrict__ pred, const uint16_t* __restrict__ labels,
                                                       const unsigned* __restrict__ invalid, unsigned long long* __restrict__ out) {
    const long long g = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int n_warps = gridDim.x * (blockDim.x >> 5);
    unsigned long long tp = 0, fp = 0, fn = 0;
    for (int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < LB2_SSC_WORDS; w += n_warps) {
        const long long gw = g * LB2_SSC_WORDS + w;
        const unsigned label = __ldg(labels + gw * 32 + lane);
        const unsigned occ = __ballot_sync(0xffffffffu, ssc_occupied(label));
        const unsigned ign = __ballot_sync(0xffffffffu, label == LB2_SSC_IGNORE);
        const unsigned p = ssc_ascending(__ldg(pred + gw));
        const unsigned valid = ~(ign | (invalid ? ssc_ascending(__ldg(invalid + gw)) : 0u));
        const unsigned gt = occ & valid;
        tp += __popc(p & gt);
        fp += __popc(p & ~gt & valid);
        fn += __popc(~p & gt);
    }
    if (lane == 0) {                                                  // every lane holds the same counts
        if (tp) atomicAdd(out + 3 * g, tp);
        if (fp) atomicAdd(out + 3 * g + 1, fp);
        if (fn) atomicAdd(out + 3 * g + 2, fn);
    }
}

// scratch: masks (uint32[G][W]), then the per-word counts / offsets (uint32[G][W]), then the grids' totals (int64[G])
extern "C" size_t lb2_ssc_scratch_bytes(int64_t n_grids) {
    return n_grids > 0 ? (size_t)n_grids * (2 * LB2_SSC_WORDS * sizeof(uint32_t) + sizeof(int64_t)) : 0;
}

extern "C" int lb2_ssc_grid_count(void* handle, void* stream, const void* grids, int32_t kind, int64_t n_grids, int64_t* offsets,
                                  void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && grids && offsets && scratch, "ssc_grid_count: null pointer");
    LB2_REQUIRE(h, kind == LB2_SSC_BITS || kind == LB2_SSC_LABELS, "ssc_grid_count: kind");
    LB2_REQUIRE(h, n_grids >= 1 && n_grids <= 4096, "ssc_grid_count: n_grids must be in [1, 4096]");
    LB2_REQUIRE(h, ((uintptr_t)scratch & 15) == 0, "ssc_grid_count: scratch must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned* masks = (unsigned*)scratch;
    unsigned* counts = masks + n_grids * LB2_SSC_WORDS;
    long long* total = (long long*)(counts + n_grids * LB2_SSC_WORDS);
    if (kind == LB2_SSC_LABELS) {
        const long long nv = n_grids * LB2_SSC_VOXELS;
        k_ssc_count_labels<<<cdiv(nv, 256), 256, 0, s>>>((const uint16_t*)grids, masks, counts);
        LB2_POST_LAUNCH(h, "k_ssc_count_labels");
    } else {
        const long long nw = n_grids * LB2_SSC_WORDS;
        k_ssc_count_bits<<<cdiv(nw, 256), 256, 0, s>>>((const unsigned*)grids, nw, masks, counts);
        LB2_POST_LAUNCH(h, "k_ssc_count_bits");
    }
    k_ssc_scan<<<(unsigned)n_grids, SSC_SCAN_THREADS, 0, s>>>(counts, total);
    LB2_POST_LAUNCH(h, "k_ssc_scan");
    k_ssc_offsets<<<1, 1, 0, s>>>(total, n_grids, (long long*)offsets);
    LB2_POST_LAUNCH(h, "k_ssc_offsets");
    return LB2_OK;
}

extern "C" int lb2_ssc_grid_points(void* handle, void* stream, int64_t n_grids, const int64_t* offsets, const void* scratch, double* out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && offsets && scratch && out, "ssc_grid_points: null pointer");
    LB2_REQUIRE(h, n_grids >= 1 && n_grids <= 4096, "ssc_grid_points: n_grids must be in [1, 4096]");
    const unsigned* masks = (const unsigned*)scratch;
    k_ssc_emit<<<cdiv(n_grids * LB2_SSC_VOXELS, 256), 256, 0, (cudaStream_t)stream>>>(masks, masks + n_grids * LB2_SSC_WORDS,
                                                                                      (const long long*)offsets, out);
    LB2_POST_LAUNCH(h, "k_ssc_emit");
    return LB2_OK;
}

extern "C" int lb2_ssc_voxelize(void* handle, void* stream, const double* pts, const int64_t* offsets, int64_t n_grids, int64_t n_points,
                                uint32_t* bits, lb2_ssc_voxel_info* d_info) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && offsets && bits && d_info && (pts || n_points == 0), "ssc_voxelize: null pointer");
    LB2_REQUIRE(h, n_grids >= 1 && n_grids <= 4096, "ssc_voxelize: n_grids must be in [1, 4096]");
    LB2_REQUIRE(h, n_points >= 0 && n_points < (1ll << 40), "ssc_voxelize: n_points");
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(bits, 0, (size_t)n_grids * LB2_SSC_WORDS * sizeof(uint32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_info, 0, (size_t)n_grids * sizeof(lb2_ssc_voxel_info), s);
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "ssc_voxelize memset: %s", cudaGetErrorString(e));
    if (n_points == 0) return LB2_OK;
    k_ssc_voxelize<<<cdiv(n_points, 256), 256, 0, s>>>(pts, (const long long*)offsets, n_grids, n_points, bits, d_info);
    LB2_POST_LAUNCH(h, "k_ssc_voxelize");
    return LB2_OK;
}

extern "C" int lb2_ssc_confusion(void* handle, void* stream, const uint32_t* pred_bits, const uint16_t* gt_labels, const uint32_t* invalid,
                                 int64_t n_grids, int64_t* out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && pred_bits && gt_labels && out, "ssc_confusion: null pointer");
    LB2_REQUIRE(h, n_grids >= 1 && n_grids <= 65535, "ssc_confusion: n_grids must be in [1, 65535]");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(out, 0, (size_t)n_grids * 3 * sizeof(int64_t), s) != cudaSuccess)
        return lb2_fail(h, LB2_ERR_CUDA, "ssc_confusion memset%s", "");
    k_ssc_confusion<<<dim3(SSC_CONF_BLOCKS, (unsigned)n_grids), 256, 0, s>>>(pred_bits, gt_labels, invalid, (unsigned long long*)out);
    LB2_POST_LAUNCH(h, "k_ssc_confusion");
    return LB2_OK;
}
