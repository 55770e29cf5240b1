// Evaluation metrics of completed scans (lidiff/utils/metrics.py:63-221, histogram_metrics.py:7-51): exact fp64 nearest-neighbour
// distances, np.histogramdd-exact voxel occupancy and counts, and deterministic reductions (integer counts, fixed-order fp64 sums).
#include <math_constants.h>
#include <algorithm>
#include "common.cuh"

// ---------------------------------------------------------------------------------------------------
// point-cloud tree: the reference cloud sorted along a Morton curve (10 bits per axis of the cubic cell grid spanning its bounding
// box), leaves of PC_LEAF consecutive sorted points, a complete binary tree in heap order whose node boxes are fp32, rounded outward
// from the fp64 bounds of their points.  The quantisation only orders the points; the search is exact in fp64 (k_pc_query).
// Buffer layout: header (bounding box as order-preserving uint64 keys [6], nleaf, n) | nodes float[2*nleaf][8] {lo xyz, 0, hi xyz, 0}
//                | sorted points double4[nleaf*PC_LEAF] (x, y, z, original index; index -1 past the last point) | build scratch.
// ---------------------------------------------------------------------------------------------------
#define PC_LEAF 8
#define PC_HDR 64                                   // bytes
#define PC_STACK 64
#define PC_BITS 10                                  // Morton bits per axis: 30-bit codes, 4 radix passes

static int pc_nleaf(int n_cap) { int n = 1; while ((long long)n * PC_LEAF < n_cap) n <<= 1; return n; }
static size_t pc_nodes_bytes(int nleaf) { return (size_t)2 * nleaf * 8 * sizeof(float); }
static size_t pc_points_bytes(int nleaf) { return (size_t)nleaf * PC_LEAF * sizeof(double4); }
static size_t pc_sort_bytes(int n_cap) { return 2 * (size_t)n_cap * sizeof(int) + rs_sort_scratch_bytes(n_cap, 3 * PC_BITS); }

extern "C" size_t lb2_pc_tree_bytes(int32_t n_cap) {
    if (n_cap <= 0) return 0;
    const int nleaf = pc_nleaf(n_cap);
    return PC_HDR + pc_nodes_bytes(nleaf) + pc_points_bytes(nleaf) + pc_sort_bytes(n_cap);
}
extern "C" size_t lb2_pc_nn_scratch_bytes(int32_t nq_cap) { return nq_cap > 0 ? pc_sort_bytes(nq_cap) : 0; }

// doubles as uint64 keys with the same order (atomicMin / atomicMax on integers: the bounding box does not depend on the order)
__device__ __forceinline__ unsigned long long pc_okey(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double pc_unkey(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__global__ void k_pc_init(unsigned long long* __restrict__ hdr, int nleaf, int n) {
    if (threadIdx.x < 3) { hdr[threadIdx.x] = ~0ull; hdr[3 + threadIdx.x] = 0ull; }
    if (threadIdx.x == 0) { int* hi = (int*)(hdr + 6); hi[0] = nleaf; hi[1] = n; }
}

__global__ void k_pc_bbox(const double* __restrict__ p, int n, unsigned long long* __restrict__ hdr) {
    unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const unsigned long long k = pc_okey(__ldg(p + 3 * (size_t)i + a));
            lo[a] = min(lo[a], k); hi[a] = max(hi[a], k);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        if ((threadIdx.x & 31) == 0) { atomicMin(hdr + a, lo[a]); atomicMax(hdr + 3 + a, hi[a]); }
    }
}

__device__ __forceinline__ unsigned pc_spread10(unsigned v) {      // 10 bits -> every third bit
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

// Morton code of each point in the cubic grid over the tree's bounding box (points outside it, i.e. queries, are clamped to its faces)
__global__ void k_pc_morton(const double* __restrict__ p, int n, const unsigned long long* __restrict__ hdr, unsigned* __restrict__ codes) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double lo[3], ext = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] = pc_unkey(hdr[a]); ext = fmax(ext, pc_unkey(hdr[3 + a]) - lo[a]); }
    const double scale = ext > 0.0 ? (double)((1 << PC_BITS) - 1) / ext : 0.0;
    unsigned c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double v = (__ldg(p + 3 * (size_t)i + a) - lo[a]) * scale;
        c[a] = (unsigned)fmin(fmax(v, 0.0), (double)((1 << PC_BITS) - 1));          // NaN -> 0
    }
    codes[i] = pc_spread10(c[0]) | (pc_spread10(c[1]) << 1) | (pc_spread10(c[2]) << 2);
}

__global__ void k_pc_gather(const double* __restrict__ p, int n, const int* __restrict__ order, int slots, double4* __restrict__ sp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    if (i >= n) { sp[i] = make_double4(0.0, 0.0, 0.0, -1.0); return; }
    const int j = order[i];
    sp[i] = make_double4(__ldg(p + 3 * (size_t)j), __ldg(p + 3 * (size_t)j + 1), __ldg(p + 3 * (size_t)j + 2), (double)j);
}

// leaf boxes: fp32 bounds rounded outward from the fp64 extremes, so every point lies inside its leaf's box; an empty leaf has lo > hi
__global__ void k_pc_leaves(const double4* __restrict__ sp, int n, int nleaf, float* __restrict__ nodes) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= nleaf) return;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int t = 0; t < PC_LEAF; ++t) {
        const int i = l * PC_LEAF + t;
        if (i >= n) break;
        const double4 q = sp[i];
        lo[0] = fmin(lo[0], q.x); lo[1] = fmin(lo[1], q.y); lo[2] = fmin(lo[2], q.z);
        hi[0] = fmax(hi[0], q.x); hi[1] = fmax(hi[1], q.y); hi[2] = fmax(hi[2], q.z);
    }
    float4* o = reinterpret_cast<float4*>(nodes + (size_t)(nleaf + l) * 8);
    o[0] = make_float4(__double2float_rd(lo[0]), __double2float_rd(lo[1]), __double2float_rd(lo[2]), 0.f);
    o[1] = make_float4(__double2float_ru(hi[0]), __double2float_ru(hi[1]), __double2float_ru(hi[2]), 0.f);
}

__global__ void __launch_bounds__(1024) k_pc_internal(int nleaf, float* __restrict__ nodes) {    // one block, level by level bottom-up
    for (int first = nleaf >> 1; first >= 1; first >>= 1) {
        for (int i = first + threadIdx.x; i < 2 * first; i += blockDim.x) {
            const float4* a = reinterpret_cast<const float4*>(nodes + (size_t)(2 * i) * 8);
            const float4 alo = a[0], ahi = a[1], blo = a[2], bhi = a[3];
            float4* o = reinterpret_cast<float4*>(nodes + (size_t)i * 8);
            o[0] = make_float4(fminf(alo.x, blo.x), fminf(alo.y, blo.y), fminf(alo.z, blo.z), 0.f);
            o[1] = make_float4(fmaxf(ahi.x, bhi.x), fmaxf(ahi.y, bhi.y), fmaxf(ahi.z, bhi.z), 0.f);
        }
        __syncthreads();
    }
}

extern "C" int lb2_pc_tree_build(void* handle, void* stream, const double* pts, int32_t n, void* tree) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && pts && tree && n > 0, "pc_tree_build");
    cudaStream_t s = (cudaStream_t)stream;
    const int nleaf = pc_nleaf(n), slots = nleaf * PC_LEAF;
    unsigned long long* hdr = (unsigned long long*)tree;
    float* nodes = (float*)((char*)tree + PC_HDR);
    double4* sp = (double4*)((char*)nodes + pc_nodes_bytes(nleaf));
    unsigned* codes = (unsigned*)((char*)sp + pc_points_bytes(nleaf));
    int* order = (int*)(codes + n);
    k_pc_init<<<1, 32, 0, s>>>(hdr, nleaf, n);
    LB2_POST_LAUNCH(h, "k_pc_init");
    k_pc_bbox<<<std::min<unsigned>(cdiv(n, 256), 264u), 256, 0, s>>>(pts, n, hdr);
    LB2_POST_LAUNCH(h, "k_pc_bbox");
    k_pc_morton<<<cdiv(n, 256), 256, 0, s>>>(pts, n, hdr, codes);
    LB2_POST_LAUNCH(h, "k_pc_morton");
    const int rc = rs_sort_keys(h, s, codes, nullptr, n, 3 * PC_BITS, order, order + n);
    if (rc != LB2_OK) return rc;
    k_pc_gather<<<cdiv(slots, 256), 256, 0, s>>>(pts, n, order, slots, sp);
    LB2_POST_LAUNCH(h, "k_pc_gather");
    k_pc_leaves<<<cdiv(nleaf, 256), 256, 0, s>>>(sp, n, nleaf, nodes);
    LB2_POST_LAUNCH(h, "k_pc_leaves");
    k_pc_internal<<<1, 1024, 0, s>>>(nleaf, nodes);
    LB2_POST_LAUNCH(h, "k_pc_internal");
    return LB2_OK;
}

// squared distance in fp64 without FMA contraction: (dx*dx + dy*dy) + dz*dz, every operation rounded on its own
__device__ __forceinline__ double pc_d2(double dx, double dy, double dz) {
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}
// lower bound of pc_d2 over the points inside a node's box: with lo <= p exactly, fl(lo - q) <= fl(p - q) (rounding is monotone),
// so the bound never exceeds the distance the leaf test computes for any point of the box.  Empty box -> +inf.
__device__ __forceinline__ double pc_box_d2(const float* __restrict__ node, double qx, double qy, double qz) {
    const float4 lo = __ldg(reinterpret_cast<const float4*>(node)), hi = __ldg(reinterpret_cast<const float4*>(node) + 1);
    if (lo.x > hi.x) return INFINITY;
    const double dx = fmax(fmax(__dsub_rn((double)lo.x, qx), __dsub_rn(qx, (double)hi.x)), 0.0);
    const double dy = fmax(fmax(__dsub_rn((double)lo.y, qy), __dsub_rn(qy, (double)hi.y)), 0.0);
    const double dz = fmax(fmax(__dsub_rn((double)lo.z, qz), __dsub_rn(qz, (double)hi.z)), 0.0);
    return pc_d2(dx, dy, dz);
}

// one thread per query, queries taken in their Morton order (order[t]) so that a warp searches one neighbourhood.  Depth-first,
// nearer child first; a subtree is skipped only when its box is strictly farther than the best point so far, so every point at the
// best distance is seen and the lowest index wins.  Cost ~O(log n) box tests per query however far the query is from the cloud.
__global__ void __launch_bounds__(128) k_pc_query(const double* __restrict__ q, int nq, const int* __restrict__ order,
                                                  const unsigned long long* __restrict__ tree, double* __restrict__ dist,
                                                  int* __restrict__ idx) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq) return;
    const int nleaf = reinterpret_cast<const int*>(tree + 6)[0];
    const float* nodes = reinterpret_cast<const float*>(reinterpret_cast<const char*>(tree) + PC_HDR);
    const double4* sp = reinterpret_cast<const double4*>(nodes + (size_t)2 * nleaf * 8);
    const int j = order[t];
    const double qx = __ldg(q + 3 * (size_t)j), qy = __ldg(q + 3 * (size_t)j + 1), qz = __ldg(q + 3 * (size_t)j + 2);
    double best = INFINITY;
    int best_i = 0x7fffffff;
    int st_node[PC_STACK];
    double st_lb[PC_STACK];
    int sp_n = 1;
    st_node[0] = 1; st_lb[0] = pc_box_d2(nodes + 8, qx, qy, qz);
    while (sp_n > 0) {
        --sp_n;
        const int node = st_node[sp_n];
        const double lb = st_lb[sp_n];
        if (lb == INFINITY || lb > best) continue;
        if (node >= nleaf) {
            const int k0 = (node - nleaf) * PC_LEAF;
#pragma unroll
            for (int u = 0; u < PC_LEAF; ++u) {
                const double2 pxy = __ldg(reinterpret_cast<const double2*>(sp + k0 + u)),
                              pzw = __ldg(reinterpret_cast<const double2*>(sp + k0 + u) + 1);
                const int pi = (int)pzw.y;
                if (pi < 0) break;                                   // padding slots are at the end of the last leaves only
                const double d = pc_d2(__dsub_rn(qx, pxy.x), __dsub_rn(qy, pxy.y), __dsub_rn(qz, pzw.x));
                if (d < best || (d == best && pi < best_i)) { best = d; best_i = pi; }
            }
        } else {
            const double l0 = pc_box_d2(nodes + (size_t)(2 * node) * 8, qx, qy, qz), l1 = pc_box_d2(nodes + (size_t)(2 * node + 1) * 8, qx, qy, qz);
            const bool first0 = l0 <= l1;                              // nearer child popped first: pushed last
            const int nf = first0 ? 2 * node + 1 : 2 * node, nn_ = first0 ? 2 * node : 2 * node + 1;
            const double lf = first0 ? l1 : l0, ln = first0 ? l0 : l1;
            if (lf != INFINITY && lf <= best && sp_n < PC_STACK) { st_node[sp_n] = nf; st_lb[sp_n] = lf; ++sp_n; }
            if (ln != INFINITY && ln <= best && sp_n < PC_STACK) { st_node[sp_n] = nn_; st_lb[sp_n] = ln; ++sp_n; }
        }
    }
    dist[j] = __dsqrt_rn(best);
    if (idx) idx[j] = best_i;
}

extern "C" int lb2_pc_nn(void* handle, void* stream, const double* q, int32_t nq, const void* tree, double* dist, int32_t* idx,
                         void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && q && tree && dist && scratch && nq > 0, "pc_nn");
    cudaStream_t s = (cudaStream_t)stream;
    const unsigned long long* hdr = (const unsigned long long*)tree;
    unsigned* codes = (unsigned*)scratch;
    int* order = (int*)(codes + nq);
    k_pc_morton<<<cdiv(nq, 256), 256, 0, s>>>(q, nq, hdr, codes);
    LB2_POST_LAUNCH(h, "k_pc_morton");
    const int rc = rs_sort_keys(h, s, codes, nullptr, nq, 3 * PC_BITS, order, order + nq);
    if (rc != LB2_OK) return rc;
    k_pc_query<<<cdiv(nq, 128), 128, 0, s>>>(q, nq, order, hdr, dist, idx);
    LB2_POST_LAUNCH(h, "k_pc_query");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// exact self-k-NN (k <= 32) over a built tree: one warp per point of the cloud, the points taken in the tree's sorted (Morton) order
// so that consecutive warps walk the same subtrees.  Lane j holds the j-th best (d², index) so far, lexicographically ordered; a
// leaf's 8 candidates are measured by lanes 0-7 at once and inserted one at a time by ballot + shuffle-up.  The walk is warp-uniform
// and depth-first, nearer child first, and skips a box only when its bound is strictly greater than the k-th distance (+inf until k
// are held), so every point tying with the k-th is seen and the (d², index) order decides.  The DFS stack also lives in the lanes:
// lane s holds slot s (the depth of a tree over int32 points is at most 28, and the stack never holds more than depth + 1 entries).
// The list starts from the 32 points around the query in the sorted order; a point the walk meets again is not inserted twice.
// Non-finite coordinates never fault: a point with a NaN or infinite coordinate does not search and only finite distances enter a
// list, so a slot nothing fills (every slot of such a point, and the slots past the number of finite points) keeps index -1, d² = +inf.
// ---------------------------------------------------------------------------------------------------
#define KNN_WARPS 4

__device__ __forceinline__ bool knn_less(double da, int ia, double db, int ib) { return da < db || (da == db && ia < ib); }

__global__ void __launch_bounds__(32 * KNN_WARPS) k_pc_knn(const unsigned long long* __restrict__ tree, int n, int k,
                                                           int* __restrict__ out_idx, double* __restrict__ out_d2) {
    const int t = blockIdx.x * KNN_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (t >= n) return;                                                  // whole warps only: t is warp-uniform
    const int nleaf = reinterpret_cast<const int*>(tree + 6)[0], tree_n = reinterpret_cast<const int*>(tree + 6)[1];
    if (tree_n != n) {                                                   // not this tree's cloud: every row is left empty
        if (lane < k) {
            out_idx[(size_t)t * k + lane] = -1;
            if (out_d2) out_d2[(size_t)t * k + lane] = INFINITY;
        }
        return;
    }
    const float* nodes = reinterpret_cast<const float*>(reinterpret_cast<const char*>(tree) + PC_HDR);
    const double4* sp = reinterpret_cast<const double4*>(nodes + (size_t)2 * nleaf * 8);
    const double4 qp = sp[t];                                            // sorted slot t < n is a real point
    const double qx = qp.x, qy = qp.y, qz = qp.z;
    const int j = (int)qp.w;
    // seed the list with the 32 points around slot t in the sorted order (Morton neighbours, mostly near): lane s measures one,
    // a bitonic sort across the lanes orders them, and the walk starts with a k-th distance that already prunes most of the tree
    double best = INFINITY;                                              // this lane's entry of the sorted list
    int best_i = 0x7fffffff;
    {
        const int a0 = n >= 32 ? min(max(t - 16, 0), n - 32) : 0;
        if (a0 + lane < n) {
            const double4 sv = sp[a0 + lane];
            const double d = pc_d2(__dsub_rn(qx, sv.x), __dsub_rn(qy, sv.y), __dsub_rn(qz, sv.z));
            if (d < INFINITY) { best = d; best_i = (int)sv.w; }             // only finite distances enter (NaN fails too)
        }
#pragma unroll
        for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                const double od = __shfl_xor_sync(0xffffffffu, best, stride);
                const int oi = __shfl_xor_sync(0xffffffffu, best_i, stride);
                const bool keep_min = ((lane & stride) == 0) == ((lane & size) == 0);
                if (keep_min ? knn_less(od, oi, best, best_i) : knn_less(best, best_i, od, oi)) { best = od; best_i = oi; }
            }
        }
    }
    double kth = __shfl_sync(0xffffffffu, best, k - 1);                  // lane k-1's distance (+inf until k are held)
    int st_node = 0;                                                     // stack slot `lane`
    double st_lb = 0.0;
    int sp_n = isfinite(qx) && isfinite(qy) && isfinite(qz) ? 1 : 0;        // a non-finite point has no neighbours
    if (lane == 0) { st_node = 1; st_lb = pc_box_d2(nodes + 8, qx, qy, qz); }
    while (sp_n > 0) {
        --sp_n;
        const int node = __shfl_sync(0xffffffffu, st_node, sp_n);
        const double lb = __shfl_sync(0xffffffffu, st_lb, sp_n);
        if (lb == INFINITY || lb > kth) continue;
        if (node >= nleaf) {
            const int k0 = (node - nleaf) * PC_LEAF;
            double d = INFINITY;
            int pi = -1;
            if (lane < PC_LEAF) {
                const double2 pxy = __ldg(reinterpret_cast<const double2*>(sp + k0 + lane)),
                              pzw = __ldg(reinterpret_cast<const double2*>(sp + k0 + lane) + 1);
                pi = (int)pzw.y;
                if (pi >= 0) d = pc_d2(__dsub_rn(qx, pxy.x), __dsub_rn(qy, pxy.y), __dsub_rn(qz, pzw.x));
            }
            const int kth_i = __shfl_sync(0xffffffffu, best_i, k - 1);
            // only finite distances enter: a NaN or infinite point is nobody's neighbour
            unsigned cand = __ballot_sync(0xffffffffu, pi >= 0 && d < INFINITY && knn_less(d, pi, kth, kth_i));
            while (cand) {
                const int c = __ffs(cand) - 1;
                cand &= cand - 1;
                const double dc = __shfl_sync(0xffffffffu, d, c);
                const int ic = __shfl_sync(0xffffffffu, pi, c);
                const double kd = __shfl_sync(0xffffffffu, best, k - 1);
                const int ki = __shfl_sync(0xffffffffu, best_i, k - 1);
                if (!knn_less(dc, ic, kd, ki)) continue;                 // the list moved on since the ballot
                if (__any_sync(0xffffffffu, best_i == ic)) continue;        // already held (a seed)
                const int pos = __popc(__ballot_sync(0xffffffffu, knn_less(best, best_i, dc, ic)));
                const double up_d = __shfl_up_sync(0xffffffffu, best, 1);
                const int up_i = __shfl_up_sync(0xffffffffu, best_i, 1);
                if (lane > pos) { best = up_d; best_i = up_i; }
                else if (lane == pos) { best = dc; best_i = ic; }
            }
            kth = __shfl_sync(0xffffffffu, best, k - 1);
        } else {
            const double l0 = pc_box_d2(nodes + (size_t)(2 * node) * 8, qx, qy, qz), l1 = pc_box_d2(nodes + (size_t)(2 * node + 1) * 8, qx, qy, qz);
            const bool first0 = l0 <= l1;                                // nearer child popped first: pushed last
            const int nf = first0 ? 2 * node + 1 : 2 * node, nn_ = first0 ? 2 * node : 2 * node + 1;
            const double lf = first0 ? l1 : l0, ln = first0 ? l0 : l1;
            if (lf != INFINITY && lf <= kth) { if (lane == sp_n) { st_node = nf; st_lb = lf; } ++sp_n; }
            if (ln != INFINITY && ln <= kth) { if (lane == sp_n) { st_node = nn_; st_lb = ln; } ++sp_n; }
        }
    }
    if (lane < k) {
        out_idx[(size_t)j * k + lane] = best_i == 0x7fffffff ? -1 : best_i;
        if (out_d2) out_d2[(size_t)j * k + lane] = best;
    }
}

extern "C" int lb2_pc_knn(void* handle, void* stream, const void* tree, int32_t n, int32_t k, int32_t* idx, double* d2) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && tree && idx && n > 0 && k >= 1, "pc_knn");
    if (k > 32) return lb2_fail(h, LB2_ERR_UNSUP, "pc_knn: k > 32 is not supported%s", "");
    const int ke = std::min(k, n);
    k_pc_knn<<<cdiv(n, KNN_WARPS), 32 * KNN_WARPS, 0, (cudaStream_t)stream>>>((const unsigned long long*)tree, n, ke, idx, d2);
    LB2_POST_LAUNCH(h, "k_pc_knn");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// PCA normals as open3d 0.17 computes them (EstimateNormals with fast_normal_computation): the one-pass cumulant covariance of the
// neighbours (ComputeCovariance) and FastEigen3x3, Geometric Tools' robust symmetric 3x3 eigensolver, for the eigenvector of the
// smallest eigenvalue; a zero result becomes (0, 0, 1).  Every operation is an explicitly rounded fp64 intrinsic evaluated in the C++
// source's left-to-right order (no FMA contraction), so the covariance is bit-exact and only acos / cos differ from a host libm.
// ---------------------------------------------------------------------------------------------------
#define RN_ADD __dadd_rn
#define RN_SUB __dsub_rn
#define RN_MUL __dmul_rn
#define RN_DIV __ddiv_rn

struct nv3 { double x, y, z; };
__device__ __forceinline__ nv3 nv_cross(nv3 a, nv3 b) {
    return {RN_SUB(RN_MUL(a.y, b.z), RN_MUL(a.z, b.y)), RN_SUB(RN_MUL(a.z, b.x), RN_MUL(a.x, b.z)), RN_SUB(RN_MUL(a.x, b.y), RN_MUL(a.y, b.x))};
}
__device__ __forceinline__ double nv_dot(nv3 a, nv3 b) { return RN_ADD(RN_ADD(RN_MUL(a.x, b.x), RN_MUL(a.y, b.y)), RN_MUL(a.z, b.z)); }
__device__ __forceinline__ nv3 nv_div(nv3 a, double s) { return {RN_DIV(a.x, s), RN_DIV(a.y, s), RN_DIV(a.z, s)}; }

// symmetric A = {a00, a01, a02, a11, a12, a22}
__device__ __forceinline__ nv3 fe_evec0(const double* A, double ev) {
    const nv3 r0 = {RN_SUB(A[0], ev), A[1], A[2]}, r1 = {A[1], RN_SUB(A[3], ev), A[4]}, r2 = {A[2], A[4], RN_SUB(A[5], ev)};
    const nv3 c01 = nv_cross(r0, r1), c02 = nv_cross(r0, r2), c12 = nv_cross(r1, r2);
    const double d0 = nv_dot(c01, c01), d1 = nv_dot(c02, c02), d2 = nv_dot(c12, c12);
    double dmax = d0;
    int imax = 0;
    if (d1 > dmax) { dmax = d1; imax = 1; }
    if (d2 > dmax) imax = 2;
    if (imax == 0) return nv_div(c01, __dsqrt_rn(d0));
    if (imax == 1) return nv_div(c02, __dsqrt_rn(d1));
    return nv_div(c12, __dsqrt_rn(d2));
}

__device__ __forceinline__ nv3 fe_evec1(const double* A, nv3 e0, double ev1) {
    nv3 U;
    if (fabs(e0.x) > fabs(e0.y)) {
        const double inv = RN_DIV(1.0, __dsqrt_rn(RN_ADD(RN_MUL(e0.x, e0.x), RN_MUL(e0.z, e0.z))));
        U = {RN_MUL(-e0.z, inv), 0.0, RN_MUL(e0.x, inv)};
    } else {
        const double inv = RN_DIV(1.0, __dsqrt_rn(RN_ADD(RN_MUL(e0.y, e0.y), RN_MUL(e0.z, e0.z))));
        U = {0.0, RN_MUL(e0.z, inv), RN_MUL(-e0.y, inv)};
    }
    const nv3 V = nv_cross(e0, U);
    const nv3 r0 = {A[0], A[1], A[2]}, r1 = {A[1], A[3], A[4]}, r2 = {A[2], A[4], A[5]};
    const nv3 AU = {nv_dot(r0, U), nv_dot(r1, U), nv_dot(r2, U)}, AV = {nv_dot(r0, V), nv_dot(r1, V), nv_dot(r2, V)};
    double m00 = RN_SUB(nv_dot(U, AU), ev1), m01 = nv_dot(U, AV), m11 = RN_SUB(nv_dot(V, AV), ev1);
    const double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
    if (a00 >= a11) {
        if (fmax(a00, a01) > 0.0) {
            if (a00 >= a01) { m01 = RN_DIV(m01, m00); m00 = RN_DIV(1.0, __dsqrt_rn(RN_ADD(1.0, RN_MUL(m01, m01)))); m01 = RN_MUL(m01, m00); }
            else { m00 = RN_DIV(m00, m01); m01 = RN_DIV(1.0, __dsqrt_rn(RN_ADD(1.0, RN_MUL(m00, m00)))); m00 = RN_MUL(m00, m01); }
            return {RN_SUB(RN_MUL(m01, U.x), RN_MUL(m00, V.x)), RN_SUB(RN_MUL(m01, U.y), RN_MUL(m00, V.y)), RN_SUB(RN_MUL(m01, U.z), RN_MUL(m00, V.z))};
        }
        return U;
    }
    if (fmax(a11, a01) > 0.0) {
        if (a11 >= a01) { m01 = RN_DIV(m01, m11); m11 = RN_DIV(1.0, __dsqrt_rn(RN_ADD(1.0, RN_MUL(m01, m01)))); m01 = RN_MUL(m01, m11); }
        else { m11 = RN_DIV(m11, m01); m01 = RN_DIV(1.0, __dsqrt_rn(RN_ADD(1.0, RN_MUL(m11, m11)))); m11 = RN_MUL(m11, m01); }
        return {RN_SUB(RN_MUL(m11, U.x), RN_MUL(m01, V.x)), RN_SUB(RN_MUL(m11, U.y), RN_MUL(m01, V.y)), RN_SUB(RN_MUL(m11, U.z), RN_MUL(m01, V.z))};
    }
    return U;
}

// FastEigen3x3 of the covariance C = {c00, c01, c02, c11, c12, c22}: eigenvector of the smallest eigenvalue, or 0 when max C == 0
__device__ __forceinline__ nv3 fast_eigen3x3(const double* C) {
    double mc = C[0];
#pragma unroll
    for (int i = 1; i < 6; ++i) mc = C[i] > mc ? C[i] : mc;
    if (mc == 0.0) return {0.0, 0.0, 0.0};
    double A[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) A[i] = RN_DIV(C[i], mc);
    const double norm = RN_ADD(RN_ADD(RN_MUL(A[1], A[1]), RN_MUL(A[2], A[2])), RN_MUL(A[4], A[4]));
    if (!(norm > 0.0)) {
        const double s00 = RN_MUL(A[0], mc), s11 = RN_MUL(A[3], mc), s22 = RN_MUL(A[5], mc);
        if (s00 < s11 && s00 < s22) return {1.0, 0.0, 0.0};
        if (s11 < s00 && s11 < s22) return {0.0, 1.0, 0.0};
        return {0.0, 0.0, 1.0};
    }
    const double q = RN_DIV(RN_ADD(RN_ADD(A[0], A[3]), A[5]), 3.0);
    const double b00 = RN_SUB(A[0], q), b11 = RN_SUB(A[3], q), b22 = RN_SUB(A[5], q);
    const double p = __dsqrt_rn(RN_DIV(RN_ADD(RN_ADD(RN_ADD(RN_MUL(b00, b00), RN_MUL(b11, b11)), RN_MUL(b22, b22)), RN_MUL(norm, 2.0)), 6.0));
    const double c00 = RN_SUB(RN_MUL(b11, b22), RN_MUL(A[4], A[4]));
    const double c01 = RN_SUB(RN_MUL(A[1], b22), RN_MUL(A[4], A[2]));
    const double c02 = RN_SUB(RN_MUL(A[1], A[4]), RN_MUL(b11, A[2]));
    const double det = RN_DIV(RN_ADD(RN_SUB(RN_MUL(b00, c00), RN_MUL(A[1], c01)), RN_MUL(A[2], c02)), RN_MUL(RN_MUL(p, p), p));
    double half_det = RN_MUL(det, 0.5);
    half_det = half_det < -1.0 ? -1.0 : half_det;                         // std::min(std::max(x, -1), 1)
    half_det = 1.0 < half_det ? 1.0 : half_det;
    const double angle = RN_DIV(acos(half_det), 3.0);
    const double beta2 = RN_MUL(cos(angle), 2.0);
    const double beta0 = RN_MUL(cos(RN_ADD(angle, 2.09439510239319549)), 2.0);
    const double beta1 = -RN_ADD(beta0, beta2);
    const double ev0 = RN_ADD(q, RN_MUL(p, beta0)), ev1 = RN_ADD(q, RN_MUL(p, beta1)), ev2 = RN_ADD(q, RN_MUL(p, beta2));
    if (half_det >= 0.0) {
        const nv3 e2 = fe_evec0(A, ev2);
        if (ev2 < ev0 && ev2 < ev1) return e2;
        const nv3 e1 = fe_evec1(A, e2, ev1);
        if (ev1 < ev0 && ev1 < ev2) return e1;
        return nv_cross(e1, e2);
    }
    const nv3 e0 = fe_evec0(A, ev0);
    if (ev0 < ev1 && ev0 < ev2) return e0;
    const nv3 e1 = fe_evec1(A, e0, ev1);
    if (ev1 < ev0 && ev1 < ev2) return e1;
    return nv_cross(e0, e1);
}

__global__ void __launch_bounds__(128) k_pc_normals(const double* __restrict__ pts, int n, const int* __restrict__ idx, int k,
                                                    double* __restrict__ normals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int* row = idx + (size_t)i * k;
    bool complete = true;                                                // every index of the row is a point of the cloud
    for (int u = 0; u < k; ++u) { const int m = __ldg(row + u); complete &= m >= 0 && m < n; }
    if (!complete) {
        normals[3 * (size_t)i] = normals[3 * (size_t)i + 1] = normals[3 * (size_t)i + 2] = CUDART_NAN;
        return;
    }
    double C[6] = {1.0, 0.0, 0.0, 1.0, 0.0, 1.0};                       // identity below 3 neighbours
    if (k >= 3) {
        double s[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int u = 0; u < k; ++u) {
            const int m = __ldg(row + u);
            const double x = __ldg(pts + 3 * (size_t)m), y = __ldg(pts + 3 * (size_t)m + 1), z = __ldg(pts + 3 * (size_t)m + 2);
            s[0] = RN_ADD(s[0], x); s[1] = RN_ADD(s[1], y); s[2] = RN_ADD(s[2], z);
            s[3] = RN_ADD(s[3], RN_MUL(x, x)); s[4] = RN_ADD(s[4], RN_MUL(x, y)); s[5] = RN_ADD(s[5], RN_MUL(x, z));
            s[6] = RN_ADD(s[6], RN_MUL(y, y)); s[7] = RN_ADD(s[7], RN_MUL(y, z)); s[8] = RN_ADD(s[8], RN_MUL(z, z));
        }
        const double cnt = (double)k;
#pragma unroll
        for (int a = 0; a < 9; ++a) s[a] = RN_DIV(s[a], cnt);
        C[0] = RN_SUB(s[3], RN_MUL(s[0], s[0])); C[3] = RN_SUB(s[6], RN_MUL(s[1], s[1])); C[5] = RN_SUB(s[8], RN_MUL(s[2], s[2]));
        C[1] = RN_SUB(s[4], RN_MUL(s[0], s[1])); C[2] = RN_SUB(s[5], RN_MUL(s[0], s[2])); C[4] = RN_SUB(s[7], RN_MUL(s[1], s[2]));
    }
    nv3 v = fast_eigen3x3(C);
    if (v.x == 0.0 && v.y == 0.0 && v.z == 0.0) v = {0.0, 0.0, 1.0};
    normals[3 * (size_t)i] = v.x; normals[3 * (size_t)i + 1] = v.y; normals[3 * (size_t)i + 2] = v.z;
}

extern "C" int lb2_pc_normals(void* handle, void* stream, const double* pts, int32_t n, const int32_t* idx, int32_t k, double* normals) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && pts && normals && n > 0 && k >= 0 && (idx || k == 0), "pc_normals");
    k_pc_normals<<<cdiv(n, 128), 128, 0, (cudaStream_t)stream>>>(pts, n, idx, k, normals);
    LB2_POST_LAUNCH(h, "k_pc_normals");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// voxel occupancy / counts with np.histogramdd's binning: bin = searchsorted(edges, x, 'right') - 1 per axis, the last edge belongs
// to the last bin, anything outside [edges[0], edges[bins]] (or NaN) is dropped.  The arithmetic guess is corrected against the fp64
// edge table, so membership is decided by the same comparisons numpy makes.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int vx_bin(double x, const double* __restrict__ e, int bins) {
    const double e0 = __ldg(e), en = __ldg(e + bins);
    if (!(x >= e0 && x <= en)) return -1;
    int g = (int)floor((x - e0) / (en - e0) * bins);
    g = min(max(g, 0), bins - 1);
    while (g > 0 && x < __ldg(e + g)) --g;
    while (g < bins - 1 && x >= __ldg(e + g + 1)) ++g;
    return g;
}

__global__ void k_vx_occupancy(const double* __restrict__ p, int n, const double* __restrict__ edges, int bins, unsigned* __restrict__ bits,
                               unsigned* __restrict__ counts, unsigned long long* __restrict__ n_in) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    bool in = false;
    if (i < n) {
        const int bx = vx_bin(__ldg(p + 3 * (size_t)i), edges, bins), by = vx_bin(__ldg(p + 3 * (size_t)i + 1), edges, bins),
                  bz = vx_bin(__ldg(p + 3 * (size_t)i + 2), edges, bins);
        in = bx >= 0 && by >= 0 && bz >= 0;
        if (in) {
            const long long cell = ((long long)bx * bins + by) * bins + bz;          // C order: x slowest, z fastest
            if (bits) atomicOr(bits + (cell >> 5), 1u << (cell & 31));
            if (counts) atomicAdd(counts + cell, 1u);
        }
    }
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (n_in && (threadIdx.x & 31) == 0 && b) atomicAdd(n_in, (unsigned long long)__popc(b));
}

extern "C" int lb2_voxel_occupancy(void* handle, void* stream, const double* pts, int32_t n, const double* edges, int32_t bins,
                                   uint32_t* bits, uint32_t* counts, uint64_t* n_in) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && pts && edges && n >= 0 && bins > 0 && bins <= 2048 && (bits || counts), "voxel_occupancy");
    cudaStream_t s = (cudaStream_t)stream;
    const long long cells = (long long)bins * bins * bins;
    cudaError_t e = cudaSuccess;
    if (bits) e = cudaMemsetAsync(bits, 0, (size_t)cdiv(cells, 32) * sizeof(uint32_t), s);
    if (e == cudaSuccess && counts) e = cudaMemsetAsync(counts, 0, (size_t)cells * sizeof(uint32_t), s);
    if (e == cudaSuccess && n_in) e = cudaMemsetAsync(n_in, 0, sizeof(uint64_t), s);
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "voxel_occupancy memset: %s", cudaGetErrorString(e));
    if (n == 0) return LB2_OK;
    k_vx_occupancy<<<cdiv(n, 256), 256, 0, s>>>(pts, n, edges, bins, bits, counts, (unsigned long long*)n_in);
    LB2_POST_LAUNCH(h, "k_vx_occupancy");
    return LB2_OK;
}

// completion IoU confusion counts of two occupancy bitsets: out = {tp = |gt & pred|, fn = |gt & ~pred|, fp = |~gt & pred|}
__global__ void k_vx_confusion(const unsigned* __restrict__ a, const unsigned* __restrict__ b, long long nwords,
                               unsigned long long* __restrict__ out) {
    unsigned long long tp = 0, fn = 0, fp = 0;
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (long long)gridDim.x * blockDim.x) {
        const unsigned x = __ldg(a + w), y = __ldg(b + w);
        tp += __popc(x & y); fn += __popc(x & ~y); fp += __popc(~x & y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tp += __shfl_xor_sync(0xffffffffu, tp, o); fn += __shfl_xor_sync(0xffffffffu, fn, o); fp += __shfl_xor_sync(0xffffffffu, fp, o);
    }
    if ((threadIdx.x & 31) == 0) { atomicAdd(out, tp); atomicAdd(out + 1, fn); atomicAdd(out + 2, fp); }
}

extern "C" int lb2_occupancy_confusion(void* handle, void* stream, const uint32_t* bits_gt, const uint32_t* bits_pred, int64_t nbits,
                                       uint64_t* out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && bits_gt && bits_pred && out && nbits > 0, "occupancy_confusion");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(out, 0, 3 * sizeof(uint64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "occupancy_confusion memset%s", "");
    const long long nwords = cdiv(nbits, 32);                    // the bits past nbits are zero in both (lb2_voxel_occupancy clears them)
    k_vx_confusion<<<std::min<unsigned>(cdiv(nwords, 256), 8 * (unsigned)h->num_sms), 256, 0, s>>>(
        (const unsigned*)bits_gt, (const unsigned*)bits_pred, nwords, (unsigned long long*)out);
    LB2_POST_LAUNCH(h, "k_vx_confusion");
    return LB2_OK;
}

// bird's-eye histogram of an occupancy: bev[x * bins + y] = number of occupied z cells of column (x, y)
__global__ void k_vx_bev(const unsigned* __restrict__ bits, int bins, unsigned* __restrict__ bev) {
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= (long long)bins * bins) return;
    const long long b0 = c * bins, b1 = b0 + bins;
    unsigned cnt = 0;
    for (long long w = b0 >> 5; w <= (b1 - 1) >> 5; ++w) {
        const int lo = (int)(max(b0, w * 32) - w * 32), hi = (int)(min(b1, w * 32 + 32) - w * 32);
        const unsigned m = (hi == 32 ? ~0u : ((1u << hi) - 1u)) & ~((1u << lo) - 1u);
        cnt += __popc(__ldg(bits + w) & m);
    }
    bev[c] = cnt;
}

extern "C" int lb2_occupancy_bev(void* handle, void* stream, const uint32_t* bits, int32_t bins, uint32_t* bev) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && bits && bev && bins > 0 && bins <= 2048, "occupancy_bev");
    k_vx_bev<<<cdiv((long long)bins * bins, 256), 256, 0, (cudaStream_t)stream>>>((const unsigned*)bits, bins, bev);
    LB2_POST_LAUNCH(h, "k_vx_bev");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// fixed-order fp64 reductions: RD_BLOCKS (or fewer) blocks of 256 threads, thread t of block b sums elements b*256 + t + k*stride in
// increasing k, the block reduces its threads by a fixed tree, one thread adds the block partials in block order.  The grid depends
// on n only, so a given input gives the same bits on every run.
// ---------------------------------------------------------------------------------------------------
#define RD_THREADS 256
#define RD_BLOCKS 1024

static unsigned rd_blocks(long long n) { return std::max(1u, std::min<unsigned>(cdiv(n, RD_THREADS), RD_BLOCKS)); }

__device__ __forceinline__ double rd_block_sum(double v, double* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = RD_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + o]);
        __syncthreads();
    }
    return sh[0];
}

__global__ void __launch_bounds__(RD_THREADS) k_sum_u32_pair(const unsigned* __restrict__ a, const unsigned* __restrict__ b, long long n,
                                                             unsigned long long* __restrict__ sums) {
    unsigned long long sa = 0, sb = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        sa += __ldg(a + i); sb += __ldg(b + i);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, o); sb += __shfl_xor_sync(0xffffffffu, sb, o); }
    if ((threadIdx.x & 31) == 0) { atomicAdd(sums, sa); atomicAdd(sums + 1, sb); }
}

// p = a / sum(a), q = b / sum(b), m = (p + q) / 2; per element rel_entr(p, m) + rel_entr(q, m) (x log(x / m), 0 where x == 0)
__global__ void __launch_bounds__(RD_THREADS) k_jsd_partial(const unsigned* __restrict__ a, const unsigned* __restrict__ b, long long n,
                                                            const unsigned long long* __restrict__ sums, double* __restrict__ partial) {
    __shared__ double sh[RD_THREADS];
    const double sa = (double)sums[0], sb = (double)sums[1];
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned ca = __ldg(a + i), cb = __ldg(b + i);
        if ((ca | cb) == 0u) continue;
        const double p = __ddiv_rn((double)ca, sa), q = __ddiv_rn((double)cb, sb);
        const double m = __dmul_rn(__dadd_rn(p, q), 0.5);
        double t = 0.0;
        if (ca) t = __dmul_rn(p, log(__ddiv_rn(p, m)));
        if (cb) t = __dadd_rn(t, __dmul_rn(q, log(__ddiv_rn(q, m))));
        acc = __dadd_rn(acc, t);
    }
    const double s = rd_block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void k_jsd_final(const double* __restrict__ partial, int nblk, const unsigned long long* __restrict__ sums, double* __restrict__ out) {
    if (threadIdx.x != 0) return;
    if (sums[0] == 0 || sums[1] == 0) { *out = CUDART_NAN; return; }
    double s = 0.0;
    for (int i = 0; i < nblk; ++i) s = __dadd_rn(s, partial[i]);
    *out = __dsqrt_rn(fmax(__dmul_rn(s, 0.5), 0.0));
}

extern "C" size_t lb2_jsd_scratch_bytes(int64_t n) { (void)n; return 2 * sizeof(uint64_t) + RD_BLOCKS * sizeof(double); }

extern "C" int lb2_jsd(void* handle, void* stream, const uint32_t* hist_a, const uint32_t* hist_b, int64_t n, double* out, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && hist_a && hist_b && out && scratch && n > 0, "jsd");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* sums = (unsigned long long*)scratch;
    double* partial = (double*)(sums + 2);
    if (cudaMemsetAsync(sums, 0, 2 * sizeof(uint64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "jsd memset%s", "");
    const unsigned nblk = rd_blocks(n);
    k_sum_u32_pair<<<nblk, RD_THREADS, 0, s>>>(hist_a, hist_b, n, sums);
    LB2_POST_LAUNCH(h, "k_sum_u32_pair");
    k_jsd_partial<<<nblk, RD_THREADS, 0, s>>>(hist_a, hist_b, n, sums, partial);
    LB2_POST_LAUNCH(h, "k_jsd_partial");
    k_jsd_final<<<1, 32, 0, s>>>(partial, (int)nblk, sums, out);
    LB2_POST_LAUNCH(h, "k_jsd_final");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// distance statistics: the fp64 sum of the distances, and for every threshold t_k (sorted ascending) the number of distances < t_k.
// Each distance lands in bin searchsorted(t, d, 'right') (the first threshold above it); counts[k] = sum of bins 0..k.
// ---------------------------------------------------------------------------------------------------
#define DS_MAX_T 4096

__global__ void __launch_bounds__(RD_THREADS) k_ds_partial(const double* __restrict__ d, int n, const double* __restrict__ thr, int nt,
                                                           double* __restrict__ partial, unsigned long long* __restrict__ hist) {
    __shared__ double sh[RD_THREADS];
    __shared__ unsigned hs[DS_MAX_T + 1];
    for (int k = threadIdx.x; k <= nt; k += blockDim.x) hs[k] = 0u;
    __syncthreads();
    double acc = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double v = __ldg(d + i);
        acc = __dadd_rn(acc, v);
        int lo = 0, hi = nt;                                     // first k with thr[k] > v
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(thr + mid) > v) hi = mid; else lo = mid + 1; }
        atomicAdd(&hs[lo], 1u);
    }
    const double s = rd_block_sum(acc, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
    for (int k = threadIdx.x; k < nt; k += blockDim.x)
        if (hs[k]) atomicAdd(hist + k, (unsigned long long)hs[k]);
}

__global__ void k_ds_final(const double* __restrict__ partial, int nblk, const unsigned long long* __restrict__ hist, int nt,
                           double* __restrict__ sum_out, unsigned long long* __restrict__ counts) {
    if (threadIdx.x != 0) return;
    double s = 0.0;
    for (int i = 0; i < nblk; ++i) s = __dadd_rn(s, partial[i]);
    *sum_out = s;
    unsigned long long run = 0;
    for (int k = 0; k < nt; ++k) { run += hist[k]; counts[k] = run; }
}

extern "C" size_t lb2_dist_stats_scratch_bytes(int32_t nt) { return (size_t)(nt + 1) * sizeof(uint64_t) + RD_BLOCKS * sizeof(double); }

extern "C" int lb2_dist_stats(void* handle, void* stream, const double* dist, int32_t n, const double* thresholds, int32_t nt,
                              double* sum_out, uint64_t* counts_out, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && dist && sum_out && scratch && n > 0 && nt >= 0 && nt <= DS_MAX_T && (nt == 0 || (thresholds && counts_out)),
                "dist_stats");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* hist = (unsigned long long*)scratch;
    double* partial = (double*)(hist + nt + 1);
    if (cudaMemsetAsync(hist, 0, (size_t)(nt + 1) * sizeof(uint64_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "dist_stats memset%s", "");
    const unsigned nblk = rd_blocks(n);
    k_ds_partial<<<nblk, RD_THREADS, 0, s>>>(dist, n, thresholds, nt, partial, hist);
    LB2_POST_LAUNCH(h, "k_ds_partial");
    k_ds_final<<<1, 32, 0, s>>>(partial, (int)nblk, hist, nt, sum_out, (unsigned long long*)counts_out);
    LB2_POST_LAUNCH(h, "k_ds_final");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// segment_sum: out[s] = sum of values[order[i]] over i in [offsets[s], offsets[s + 1]), added in ascending i (one warp per segment,
// lanes over channels).  The backward of a row gather (the Chamfer loss' x[idx], slice()) without atomics.
// ---------------------------------------------------------------------------------------------------
template <class T>
__global__ void k_segment_sum(const T* __restrict__ values, const int64_t* __restrict__ order, const int64_t* __restrict__ offsets,
                              int64_t nseg, int32_t c, T* __restrict__ out) {
    const int64_t seg = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (seg >= nseg) return;
    const int64_t b = offsets[seg], e = offsets[seg + 1];
    for (int j = lane; j < c; j += 32) {
        T s = 0;
        for (int64_t i = b; i < e; ++i) s += values[(order ? order[i] : i) * c + j];
        out[seg * c + j] = s;
    }
}

extern "C" int lb2_segment_sum(void* handle, void* stream, const void* values, int32_t f64, const int64_t* order,
                               const int64_t* offsets, int64_t nseg, int32_t c, void* out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && values && offsets && out && nseg >= 0 && c > 0, "segment_sum");
    if (nseg == 0) return LB2_OK;
    const unsigned grid = cdiv(nseg * 32, 256);
    if (f64) k_segment_sum<double><<<grid, 256, 0, (cudaStream_t)stream>>>((const double*)values, order, offsets, nseg, c, (double*)out);
    else k_segment_sum<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)values, order, offsets, nseg, c, (float*)out);
    LB2_POST_LAUNCH(h, "k_segment_sum");
    return LB2_OK;
}
