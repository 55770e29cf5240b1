// Uniform surface sampling of triangle meshes (lidiff/utils/metrics.py:37's geom.sample_points_uniformly, lidiff_b200/mesh.py):
// open3d 0.17's TriangleMesh::SamplePointsUniformly restated in the order of include/lidiff_b200.h, every fp64 operation rounded on
// its own so that tests/mesh_reference.py reproduces the points bit for bit.
//   * k_mesh_areas: one thread per triangle; index and finiteness violations go into the status word.
//   * k_mesh_chain: S and the cdf are sequential fp64 chains (a parallel scan rounds differently).  One warp: the 32 lanes load a
//     tile of 8 x 32 values coalesced while the previous tile is consumed, and every lane adds the tile's values in order, each
//     broadcast by a shuffle, so the only dependent instruction per value is one add.  The quotients area_t / S are independent and
//     come from a grid-wide launch in between (k_mesh_divide).
//   * k_mesh_counts: n_t = round(cdf_t N), one thread per triangle.
//   * k_mesh_sample: one thread per point: a binary search of the n_t and one uint4 of MT19937 words.
#include "common.cuh"

#define RN_ADD __dadd_rn
#define RN_SUB __dsub_rn
#define RN_MUL __dmul_rn
#define RN_DIV __ddiv_rn

#define CHAIN_ROWS 8
#define CHAIN_TILE (CHAIN_ROWS * 32)

__global__ void __launch_bounds__(256) k_mesh_areas(const double* __restrict__ verts, int64_t n_verts, const int* __restrict__ tris,
                                                    int64_t n_tris, double* __restrict__ area, lb2_mesh_info* __restrict__ info) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tris) return;
    const int i0 = __ldg(tris + 3 * t), i1 = __ldg(tris + 3 * t + 1), i2 = __ldg(tris + 3 * t + 2);
    if (i0 < 0 || i0 >= n_verts || i1 < 0 || i1 >= n_verts || i2 < 0 || i2 >= n_verts) {
        area[t] = 0.0;
        atomicOr(&info->status, LB2_MESH_BAD_INDEX);
        return;
    }
    const double* p0 = verts + 3 * (int64_t)i0;
    const double* p1 = verts + 3 * (int64_t)i1;
    const double* p2 = verts + 3 * (int64_t)i2;
    double v[9];
#pragma unroll
    for (int k = 0; k < 3; ++k) { v[k] = __ldg(p0 + k); v[3 + k] = __ldg(p1 + k); v[6 + k] = __ldg(p2 + k); }
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 9; ++k) finite &= isfinite(v[k]);
    if (!finite) atomicOr(&info->status, LB2_MESH_NON_FINITE);
    const double x0 = RN_SUB(v[0], v[3]), x1 = RN_SUB(v[1], v[4]), x2 = RN_SUB(v[2], v[5]);    // x = p0 - p1
    const double y0 = RN_SUB(v[0], v[6]), y1 = RN_SUB(v[1], v[7]), y2 = RN_SUB(v[2], v[8]);    // y = p0 - p2
    const double c0 = RN_SUB(RN_MUL(x1, y2), RN_MUL(x2, y1));
    const double c1 = RN_SUB(RN_MUL(x2, y0), RN_MUL(x0, y2));
    const double c2 = RN_SUB(RN_MUL(x0, y1), RN_MUL(x1, y0));
    area[t] = RN_MUL(0.5, __dsqrt_rn(RN_ADD(RN_ADD(RN_MUL(c0, c0), RN_MUL(c1, c1)), RN_MUL(c2, c2))));
}

// kCdf = false: info->surface_area = in[0] + in[1] + ... left to right (status LB2_MESH_BAD_AREA unless it is positive and finite);
// kCdf = true: out[t] = in[t] + out[t - 1] (out[0] = in[0]), skipped when S is bad.  One warp.
template <bool kCdf>
__global__ void __launch_bounds__(32) k_mesh_chain(const double* __restrict__ in, double* __restrict__ out, int64_t n,
                                                   lb2_mesh_info* __restrict__ info) {
    if (kCdf && (info->status & LB2_MESH_BAD_AREA)) return;
    const int lane = threadIdx.x;
    double cur[CHAIN_ROWS], nxt[CHAIN_ROWS];
#pragma unroll
    for (int j = 0; j < CHAIN_ROWS; ++j) {
        const int64_t k = j * 32 + lane;
        cur[j] = k < n ? __ldg(in + k) : 0.0;
    }
    double c = 0.0;
    for (int64_t base = 0; base < n; base += CHAIN_TILE) {
#pragma unroll
        for (int j = 0; j < CHAIN_ROWS; ++j) {                          // the next tile's loads fly while this tile is added
            const int64_t k = base + CHAIN_TILE + j * 32 + lane;
            nxt[j] = k < n ? __ldg(in + k) : 0.0;
        }
        const bool full = base + CHAIN_TILE <= n;
#pragma unroll
        for (int j = 0; j < CHAIN_ROWS; ++j) {
            double mine = 0.0;
#pragma unroll
            for (int l = 0; l < 32; ++l) {
                const double v = __shfl_sync(0xffffffffu, cur[j], l);
                if (full || base + j * 32 + l < n) c = RN_ADD(c, v);      // the same value in every lane
                if (l == lane) mine = c;
            }
            const int64_t k = base + j * 32 + lane;
            if (kCdf && k < n) out[k] = mine;
        }
#pragma unroll
        for (int j = 0; j < CHAIN_ROWS; ++j) cur[j] = nxt[j];
    }
    if (!kCdf && lane == 0) {
        info->surface_area = c;
        if (!(c > 0.0 && c <= 1.7976931348623157e308)) info->status |= LB2_MESH_BAD_AREA;
    }
}

__global__ void __launch_bounds__(256) k_mesh_divide(const double* __restrict__ area, int64_t n_tris, const lb2_mesh_info* __restrict__ info,
                                                     double* __restrict__ q) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tris || (info->status & LB2_MESH_BAD_AREA)) return;
    q[t] = RN_DIV(area[t], info->surface_area);
}

__global__ void __launch_bounds__(256) k_mesh_counts(const double* __restrict__ cdf, int64_t n_tris, int64_t n_points,
                                                     long long* __restrict__ counts, lb2_mesh_info* __restrict__ info) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tris || (info->status & LB2_MESH_BAD_AREA)) return;
    const long long n_t = (long long)round(RN_MUL(cdf[t], (double)n_points));    // round: half away from zero
    counts[t] = n_t;
    if (t == n_tris - 1) {
        info->last_count = n_t;
        if (n_t != n_points) atomicOr(&info->status, LB2_MESH_BAD_COUNT);
    }
}

// libstdc++'s generate_canonical<double, 53> over two std::mt19937 words
__device__ __forceinline__ double mesh_canonical(uint32_t lo, uint32_t hi) {
    const double r = RN_MUL(RN_ADD((double)lo, RN_MUL((double)hi, 0x1p32)), 0x1p-64);
    return r >= 1.0 ? __longlong_as_double(0x3FEFFFFFFFFFFFFFll) : r;                 // nextafter(1, 0)
}

__global__ void __launch_bounds__(256) k_mesh_sample(const double* __restrict__ verts, const int* __restrict__ tris,
                                                     const long long* __restrict__ counts, int64_t n_tris, const uint4* __restrict__ words,
                                                     int64_t n, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t lo = 0, hi = n_tris - 1;                                   // the first t with counts[t] > i (counts[n_tris - 1] == n)
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(counts + mid) > i) hi = mid; else lo = mid + 1;
    }
    const uint4 w = __ldg(words + i);
    const double r1 = mesh_canonical(w.x, w.y), r2 = mesh_canonical(w.z, w.w);
    const double s = __dsqrt_rn(r1);
    const double a = RN_SUB(1.0, s), b = RN_MUL(s, RN_SUB(1.0, r2)), c = RN_MUL(s, r2);
    const double* p0 = verts + 3 * (int64_t)__ldg(tris + 3 * lo);
    const double* p1 = verts + 3 * (int64_t)__ldg(tris + 3 * lo + 1);
    const double* p2 = verts + 3 * (int64_t)__ldg(tris + 3 * lo + 2);
#pragma unroll
    for (int k = 0; k < 3; ++k)
        out[3 * i + k] = RN_ADD(RN_ADD(RN_MUL(a, __ldg(p0 + k)), RN_MUL(b, __ldg(p1 + k))), RN_MUL(c, __ldg(p2 + k)));
}

// scratch: counts (int64[n_tris]) at 0, then the quotients and the cdf (fp64[n_tris] each)
extern "C" size_t lb2_mesh_sample_scratch_bytes(int64_t n_tris) { return (size_t)(n_tris > 0 ? n_tris : 0) * 24; }

extern "C" int lb2_mesh_sample_prepare(void* handle, void* stream, const double* verts, int64_t n_verts, const int32_t* tris, int64_t n_tris,
                                       int64_t n_points, double* area, lb2_mesh_info* d_info, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && verts && tris && area && d_info && scratch, "mesh_sample_prepare: null pointer");
    LB2_REQUIRE(h, n_verts >= 1 && n_tris >= 1, "mesh_sample_prepare: the mesh needs vertices and triangles");
    LB2_REQUIRE(h, n_points >= 1 && n_points < (1ll << 53), "mesh_sample_prepare: n_points must be in [1, 2^53)");
    LB2_REQUIRE(h, ((uintptr_t)scratch & 15) == 0, "mesh_sample_prepare: scratch must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    long long* counts = (long long*)scratch;
    double* q = (double*)scratch + n_tris;
    double* cdf = q + n_tris;
    if (cudaMemsetAsync(d_info, 0, sizeof(lb2_mesh_info), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "mesh_sample_prepare: memset");
    const unsigned grid = cdiv(n_tris, 256);
    k_mesh_areas<<<grid, 256, 0, s>>>(verts, n_verts, tris, n_tris, area, d_info);
    LB2_POST_LAUNCH(h, "k_mesh_areas");
    k_mesh_chain<false><<<1, 32, 0, s>>>(area, nullptr, n_tris, d_info);
    LB2_POST_LAUNCH(h, "k_mesh_chain<sum>");
    k_mesh_divide<<<grid, 256, 0, s>>>(area, n_tris, d_info, q);
    LB2_POST_LAUNCH(h, "k_mesh_divide");
    k_mesh_chain<true><<<1, 32, 0, s>>>(q, cdf, n_tris, d_info);
    LB2_POST_LAUNCH(h, "k_mesh_chain<cdf>");
    k_mesh_counts<<<grid, 256, 0, s>>>(cdf, n_tris, n_points, counts, d_info);
    LB2_POST_LAUNCH(h, "k_mesh_counts");
    return LB2_OK;
}

extern "C" int lb2_mesh_sample_points(void* handle, void* stream, const double* verts, const int32_t* tris, int64_t n_tris, const void* scratch,
                                      const uint32_t* words, int64_t n_points, double* out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && verts && tris && scratch && words && out, "mesh_sample_points: null pointer");
    LB2_REQUIRE(h, n_tris >= 1 && n_points >= 1 && n_points < (1ll << 53), "mesh_sample_points: sizes");
    LB2_REQUIRE(h, ((uintptr_t)words & 15) == 0, "mesh_sample_points: words must be 16-byte aligned");
    k_mesh_sample<<<cdiv(n_points, 256), 256, 0, (cudaStream_t)stream>>>(verts, tris, (const long long*)scratch, n_tris,
                                                                         (const uint4*)words, n_points, out);
    LB2_POST_LAUNCH(h, "k_mesh_sample");
    return LB2_OK;
}
