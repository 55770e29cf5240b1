// K5/K6/K7 + FPS — the non-convolution kernels of the hot path.
//   lb2_nn_match            exact 1-NN of voxel coordinates (pykeops argKmin, minkunet.py:403-418)
//   lb2_linear              torch.nn.Linear (+LeakyReLU/tanh) of the gate / head MLPs (minkunet.py:165-181,376-380)
//   lb2_gate_mul            x * w[idx]   (minkunet.py:431 ...)
//   lb2_gather_rows         F[idx]       (minkunet.py:418,497)
//   lb2_guidance_dpm_step   guidance + DPM-Solver++(2M) SDE + re-quantise (pipeline:153,162-164)
//   lb2_farthest_point_sample  open3d FPS (pipeline:97-99)
#include "common.cuh"
#include <float.h>
#include <algorithm>
#include <cooperative_groups.h>
#include "tc_common.cuh"

// ---------------------------------------------------------------------------------------------------
// nn_match: brute force, keys staged through shared memory, exact 64-bit integer distances
// ---------------------------------------------------------------------------------------------------
#define NN_THREADS 256
#define NN_KEYS    1024

__global__ void __launch_bounds__(NN_THREADS) k_nn_match(const int4* __restrict__ q, const int* __restrict__ d_nq, int nq_cap,
                                                          const int4* __restrict__ keys, const int* __restrict__ d_nk, int nk_cap,
                                                          long long batch_scale, int* __restrict__ idx) {
    __shared__ int4 ks[NN_KEYS];
    const int nq = d_nq ? min(*d_nq, nq_cap) : nq_cap;
    const int nk = d_nk ? min(*d_nk, nk_cap) : nk_cap;
    if (blockIdx.x * NN_THREADS >= nq) return;
    const int i = blockIdx.x * NN_THREADS + threadIdx.x;
    int4 c = make_int4(0, 0, 0, 0);
    if (i < nq) c = __ldg(q + i);
    unsigned long long best = ~0ull;
    int best_j = 0;
    for (int j0 = 0; j0 < nk; j0 += NN_KEYS) {
        const int cnt = min(NN_KEYS, nk - j0);
        __syncthreads();
        for (int j = threadIdx.x; j < cnt; j += NN_THREADS) ks[j] = __ldg(keys + j0 + j);
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < cnt; ++j) {
            const int4 kc = ks[j];
            const long long dx = c.y - kc.y, dy = c.z - kc.z, dz = c.w - kc.w;
            unsigned long long d = (unsigned long long)(dx * dx + dy * dy + dz * dz);
            if (c.x != kc.x) {
                if (batch_scale > 0) { long long db = (long long)(c.x - kc.x) * batch_scale; d += (unsigned long long)(db * db); }
                else d += 1ull << 62;
            }
            if (d < best) { best = d; best_j = j0 + j; }     // strict '<' => lowest index on ties
        }
    }
    if (i < nq) idx[i] = best_j;
}

extern "C" int lb2_nn_match(void* handle, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                            const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, int32_t batch_scale,
                            int32_t* idx) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && q_coords && k_coords && idx && nq_cap > 0 && nk_cap > 0, "nn_match");
    k_nn_match<<<cdiv(nq_cap, NN_THREADS), NN_THREADS, 0, (cudaStream_t)stream>>>(
        (const int4*)q_coords, d_nq, nq_cap, (const int4*)k_coords, d_nk, nk_cap, (long long)batch_scale, idx);
    LB2_POST_LAUNCH(h, "k_nn_match");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// nn_match, grid-accelerated: the keys are voxels on a lattice of pitch `ks` (the stride-16 partial-scan
// level) that already own a hash grid (coordinate -> row).  Each query walks the lattice in growing cube
// shells around its nearest lattice cell; every key outside shell r is at least ks*(r+0.5) away along one
// axis, so the search stops as soon as the best squared distance is strictly below ks^2*(r+0.5)^2 (strict:
// an equal-distance key further out could still win the lowest-index tie rule).  Same result as the brute
// force kernel, ~50x fewer distance evaluations for queries near the scan; a query that is not settled
// after `max_ring` shells falls back to the exhaustive scan.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int floor_div(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }

__global__ void __launch_bounds__(256) k_nn_match_grid(const int4* __restrict__ q, const int* __restrict__ d_nq, int nq_cap,
                                                       const int4* __restrict__ keys, const int* __restrict__ d_nk, int nk_cap,
                                                       const unsigned long long* __restrict__ gkeys, const int* __restrict__ grows, unsigned gmask,
                                                       int ks, int max_ring, int* __restrict__ idx) {
    const int nq = d_nq ? min(*d_nq, nq_cap) : nq_cap;
    const int nk = d_nk ? min(*d_nk, nk_cap) : nk_cap;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (blockIdx.x * blockDim.x >= nq) return;                       // whole block idle
    const bool live = i < nq;
    const int4 c = live ? __ldg(q + i) : make_int4(0, 0, 0, 0);
    const int cx = floor_div(c.y + ks / 2, ks), cy = floor_div(c.z + ks / 2, ks), cz = floor_div(c.w + ks / 2, ks);
    unsigned long long best = ~0ull;
    int best_j = 0x7fffffff;
    bool settled = !live;
    for (int r = 0; r <= max_ring && !settled; ++r) {
        for (int dz = -r; dz <= r; ++dz) {
            for (int dy = -r; dy <= r; ++dy) {
                const bool face = (abs(dz) == r) || (abs(dy) == r);
                const int step = face ? 1 : max(2 * r, 1);
                for (int dx = -r; dx <= r; dx += step) {
                    const int kx = (cx + dx) * ks, ky = (cy + dy) * ks, kz = (cz + dz) * ks;
                    unsigned long long key;
                    if (!lb2_pack_key(c.x, kx, ky, kz, key)) continue;
                    const int j = lb2_grid_lookup(gkeys, grows, gmask, key);
                    if (j < 0) continue;
                    const long long ex = c.y - kx, ey = c.z - ky, ez = c.w - kz;
                    const unsigned long long d = (unsigned long long)(ex * ex + ey * ey + ez * ez);
                    if (d < best || (d == best && j < best_j)) { best = d; best_j = j; }
                }
            }
        }
        const unsigned long long bound = (unsigned long long)ks * ks * (2 * r + 1) * (2 * r + 1);   // 4 * ks^2 (r+0.5)^2
        settled = (best != ~0ull) && (4ull * best < bound);
    }
    // queries far from every key: exhaustive scan, one query at a time with the whole warp (identical tie rule)
    unsigned pending = __ballot_sync(0xffffffffu, !settled);
    const int lane = threadIdx.x & 31;
    while (pending) {
        const int src = __ffs(pending) - 1;
        pending &= pending - 1;
        const int qb = __shfl_sync(0xffffffffu, c.x, src), qx = __shfl_sync(0xffffffffu, c.y, src);
        const int qy = __shfl_sync(0xffffffffu, c.z, src), qz = __shfl_sync(0xffffffffu, c.w, src);
        unsigned long long bd = ~0ull;
        int bj = 0x7fffffff;
        for (int j = lane; j < nk; j += 32) {
            const int4 kc = __ldg(keys + j);
            const long long ex = qx - kc.y, ey = qy - kc.z, ez = qz - kc.w;
            unsigned long long d = (unsigned long long)(ex * ex + ey * ey + ez * ez);
            if (qb != kc.x) d += 1ull << 62;
            if (d < bd) { bd = d; bj = j; }                          // ascending j per lane: lowest index kept
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long od = __shfl_xor_sync(0xffffffffu, bd, o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (od < bd || (od == bd && oj < bj)) { bd = od; bj = oj; }
        }
        if (lane == src) best_j = (bj == 0x7fffffff) ? 0 : bj;
    }
    if (live) idx[i] = best_j;
}

extern "C" int lb2_nn_match_grid(void* handle, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                                 const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, lb2_grid key_grid,
                                 int32_t key_stride, int32_t max_ring, int32_t* idx) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && q_coords && k_coords && idx && key_grid.keys && key_grid.vals && nq_cap > 0 && nk_cap > 0, "nn_match_grid");
    LB2_REQUIRE(h, key_stride > 0 && key_stride % 2 == 0 && max_ring >= 0 && max_ring <= 16, "nn_match_grid stride/ring");
    k_nn_match_grid<<<cdiv(nq_cap, 256), 256, 0, (cudaStream_t)stream>>>(
        (const int4*)q_coords, d_nq, nq_cap, (const int4*)k_coords, d_nk, nk_cap, (const unsigned long long*)key_grid.keys,
        key_grid.vals + key_grid.cap_table, (unsigned)key_grid.cap_table - 1u, key_stride, max_ring, idx);
    LB2_POST_LAUNCH(h, "k_nn_match_grid");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// nn_match on the bounding-volume hierarchy of lb2_nn_tree_build (coords.cu): depth-first search with the nearer
// child first, a subtree is skipped when its box is strictly farther than the best key so far ('<=' keeps equal
// distances: the lowest original row must win ties, exactly as in the exhaustive kernel).
// ---------------------------------------------------------------------------------------------------
#define NT_LEAF 4
#define NT_HDR 16
#define NT_STACK 48

// squared length of an integer offset whose components fit 32 bits (coordinates are 18-bit signed): three 32 x 32 -> 64 bit multiplies
__device__ __forceinline__ unsigned long long nt_sq3(int ex, int ey, int ez) {
    const unsigned ax = (unsigned)abs(ex), ay = (unsigned)abs(ey), az = (unsigned)abs(ez);
    return (unsigned long long)ax * ax + (unsigned long long)ay * ay + (unsigned long long)az * az;
}
__device__ __forceinline__ unsigned long long nt_box_dist(const int* __restrict__ n, const int4 c) {
    const int4 lo = __ldg(reinterpret_cast<const int4*>(n)), hi = __ldg(reinterpret_cast<const int4*>(n) + 1);   // {min xyz, max x} {max yz, batch lo, hi}
    if (lo.x > lo.w) return ~0ull;                                   // empty node
    const int dx = max(max(lo.x - c.y, c.y - lo.w), 0), dy = max(max(lo.y - c.z, c.z - hi.x), 0), dz = max(max(lo.z - c.w, c.w - hi.y), 0);
    unsigned long long d = nt_sq3(dx, dy, dz);
    if (c.x < hi.z || c.x > hi.w) d += 1ull << 62;                   // no key of the query's batch in this subtree
    return d;
}

__global__ void __launch_bounds__(128) k_nn_match_tree(const int4* __restrict__ q, const int* __restrict__ d_nq, int nq_cap,
                                                       const int* __restrict__ tree, int nk_cap, const int4* __restrict__ keys,
                                                       const int* __restrict__ hint_of, const int* __restrict__ hint_idx,
                                                       int* __restrict__ idx) {
    const int nq = d_nq ? min(*d_nq, nq_cap) : nq_cap;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const int nleaf = tree[7];
    const int* nodes = tree + NT_HDR;
    const int4* skeys = reinterpret_cast<const int4*>(nodes + (size_t)2 * nleaf * 8);
    const int* sbatch = reinterpret_cast<const int*>(skeys + (size_t)nleaf * NT_LEAF);
    const int4 c = __ldg(q + i);
    unsigned long long best = ~0ull;
    int best_j = 0x7fffffff;
    if (hint_idx) {                                                  // start from a key that is probably close (a coarser voxel's answer):
        const int j = __ldg(hint_idx + (hint_of ? __ldg(hint_of + i) : i));    // any key is a valid upper bound, so the result is unchanged
        const int4 kc = __ldg(keys + j);
        best = nt_sq3(c.y - kc.y, c.z - kc.z, c.w - kc.w);
        if (kc.x != c.x) best += 1ull << 62;
        best_j = j;
    }
    int st_node[NT_STACK];
    unsigned long long st_lb[NT_STACK];
    int sp = 0;
    st_node[0] = 1; st_lb[0] = nt_box_dist(nodes + 8, c); sp = 1;
    while (sp > 0) {
        --sp;
        const int node = st_node[sp];
        const unsigned long long lb = st_lb[sp];
        if (lb == ~0ull || lb > best) continue;
        if (node >= nleaf) {
            const int k0 = (node - nleaf) * NT_LEAF;
#pragma unroll
            for (int t = 0; t < NT_LEAF; ++t) {
                const int4 kc = __ldg(skeys + k0 + t);
                const int kb = __ldg(sbatch + k0 + t);
                unsigned long long d = nt_sq3(c.y - kc.x, c.z - kc.y, c.w - kc.z);
                if (kb != c.x) d += 1ull << 62;
                const bool valid = kc.w >= 0;                          // slots past the last key hold row -1
                if (valid && (d < best || (d == best && kc.w < best_j))) { best = d; best_j = kc.w; }
            }
        } else {
            const unsigned long long l0 = nt_box_dist(nodes + (size_t)(2 * node) * 8, c), l1 = nt_box_dist(nodes + (size_t)(2 * node + 1) * 8, c);
            const bool first0 = l0 <= l1;                              // visit the nearer child first: push it last
            const int nf = first0 ? 2 * node + 1 : 2 * node, nn_ = first0 ? 2 * node : 2 * node + 1;
            const unsigned long long lf = first0 ? l1 : l0, ln = first0 ? l0 : l1;
            if (lf != ~0ull && lf <= best && sp < NT_STACK) { st_node[sp] = nf; st_lb[sp] = lf; ++sp; }
            if (ln != ~0ull && ln <= best && sp < NT_STACK) { st_node[sp] = nn_; st_lb[sp] = ln; ++sp; }
        }
    }
    idx[i] = (best_j == 0x7fffffff) ? 0 : best_j;
}

extern "C" int lb2_nn_match_tree(void* handle, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                                 const void* tree, int32_t nk_cap, const int32_t* k_coords, const int32_t* hint_of,
                                 const int32_t* hint_idx, int32_t* idx) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && q_coords && tree && idx && nq_cap > 0 && nk_cap > 0 && (!hint_idx || k_coords), "nn_match_tree");
    k_nn_match_tree<<<cdiv(nq_cap, 128), 128, 0, (cudaStream_t)stream>>>((const int4*)q_coords, d_nq, nq_cap, (const int*)tree, nk_cap,
                                                                         (const int4*)k_coords, hint_of, hint_idx, idx);
    LB2_POST_LAUNCH(h, "k_nn_match_tree");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// nn_match with the key lattice in SHARED memory: the <= 8192 keys of the partial scan are re-hashed once per scan
// into a compact 16384-slot table (128 KB keys + 64 KB rows) that every CTA copies into its shared memory, so the
// 27-125 probes of a query are smem accesses instead of L2 round trips.  Same shell search and tie rule as above.
// ---------------------------------------------------------------------------------------------------
#define NNT_SLOTS 16384
#define NNT_THREADS 1024

__global__ void k_nn_table_build(const int4* __restrict__ keys, const int* __restrict__ d_nk, int nk_cap,
                                 unsigned long long* __restrict__ tkeys, int* __restrict__ trows, int* __restrict__ overflow) {
    const int nk = d_nk ? min(*d_nk, nk_cap) : nk_cap;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) *overflow = (nk > NNT_SLOTS / 2) ? 1 : 0;
    if (j >= nk || nk > NNT_SLOTS / 2) return;
    const int4 c = __ldg(keys + j);
    unsigned long long key;
    if (!lb2_pack_key(c.x, c.y, c.z, c.w, key)) return;            // out-of-range keys can never be probed
    unsigned slot = lb2_hash(key) & (NNT_SLOTS - 1);
    while (true) {
        const unsigned long long prev = atomicCAS(tkeys + slot, (unsigned long long)LB2_KEY_EMPTY, key);
        if (prev == LB2_KEY_EMPTY || prev == key) break;
        slot = (slot + 1) & (NNT_SLOTS - 1);
    }
    atomicMin(trows + slot, j);                                    // duplicate coordinates: lowest row wins (tie rule)
}

__global__ void __launch_bounds__(NNT_THREADS, 1) k_nn_match_table(const int4* __restrict__ q, const int* __restrict__ d_nq, int nq_cap,
                                                                   const int4* __restrict__ keys, const int* __restrict__ d_nk, int nk_cap,
                                                                   const unsigned long long* __restrict__ tkeys, const int* __restrict__ trows,
                                                                   int ks, int max_ring, int* __restrict__ idx) {
    extern __shared__ unsigned char nnt_smem[];
    unsigned long long* sk = reinterpret_cast<unsigned long long*>(nnt_smem);
    int* sr = reinterpret_cast<int*>(sk + NNT_SLOTS);
    for (int i = threadIdx.x; i < NNT_SLOTS / 2; i += NNT_THREADS) reinterpret_cast<ulonglong2*>(sk)[i] = __ldg(reinterpret_cast<const ulonglong2*>(tkeys) + i);
    for (int i = threadIdx.x; i < NNT_SLOTS / 4; i += NNT_THREADS) reinterpret_cast<int4*>(sr)[i] = __ldg(reinterpret_cast<const int4*>(trows) + i);
    __syncthreads();
    const int nq = d_nq ? min(*d_nq, nq_cap) : nq_cap;
    const int nk = d_nk ? min(*d_nk, nk_cap) : nk_cap;
    const int lane = threadIdx.x & 31;
    for (int i0 = blockIdx.x * NNT_THREADS; i0 < nq; i0 += gridDim.x * NNT_THREADS) {
        const int i = i0 + threadIdx.x;
        const bool live = i < nq;
        const int4 c = live ? __ldg(q + i) : make_int4(0, 0, 0, 0);
        const int cx = floor_div(c.y + ks / 2, ks), cy = floor_div(c.z + ks / 2, ks), cz = floor_div(c.w + ks / 2, ks);
        unsigned long long best = ~0ull;
        int best_j = 0x7fffffff;
        bool settled = !live;
        for (int r = 0; r <= max_ring && !settled; ++r) {
            for (int dz = -r; dz <= r; ++dz) {
                for (int dy = -r; dy <= r; ++dy) {
                    const bool face = (abs(dz) == r) || (abs(dy) == r);
                    const int step = face ? 1 : max(2 * r, 1);
                    for (int dx = -r; dx <= r; dx += step) {
                        const int kx = (cx + dx) * ks, ky = (cy + dy) * ks, kz = (cz + dz) * ks;
                        unsigned long long key;
                        if (!lb2_pack_key(c.x, kx, ky, kz, key)) continue;
                        unsigned slot = lb2_hash(key) & (NNT_SLOTS - 1);
                        int j = -1;
                        while (true) {
                            const unsigned long long kk = sk[slot];
                            if (kk == key) { j = sr[slot]; break; }
                            if (kk == LB2_KEY_EMPTY) break;
                            slot = (slot + 1) & (NNT_SLOTS - 1);
                        }
                        if (j < 0) continue;
                        const long long ex = c.y - kx, ey = c.z - ky, ez = c.w - kz;
                        const unsigned long long d = (unsigned long long)(ex * ex + ey * ey + ez * ez);
                        if (d < best || (d == best && j < best_j)) { best = d; best_j = j; }
                    }
                }
            }
            const unsigned long long bound = (unsigned long long)ks * ks * (2 * r + 1) * (2 * r + 1);
            settled = (best != ~0ull) && (4ull * best < bound);
        }
        unsigned pending = __ballot_sync(0xffffffffu, !settled);
        while (pending) {
            const int src = __ffs(pending) - 1;
            pending &= pending - 1;
            const int qb = __shfl_sync(0xffffffffu, c.x, src), qx = __shfl_sync(0xffffffffu, c.y, src);
            const int qy = __shfl_sync(0xffffffffu, c.z, src), qz = __shfl_sync(0xffffffffu, c.w, src);
            unsigned long long bd = ~0ull;
            int bj = 0x7fffffff;
            for (int j = lane; j < nk; j += 32) {
                const int4 kc = __ldg(keys + j);
                const long long ex = qx - kc.y, ey = qy - kc.z, ez = qz - kc.w;
                unsigned long long d = (unsigned long long)(ex * ex + ey * ey + ez * ez);
                if (qb != kc.x) d += 1ull << 62;
                if (d < bd) { bd = d; bj = j; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long od = __shfl_xor_sync(0xffffffffu, bd, o);
                const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
                if (od < bd || (od == bd && oj < bj)) { bd = od; bj = oj; }
            }
            if (lane == src) best_j = (bj == 0x7fffffff) ? 0 : bj;
        }
        if (live) idx[i] = best_j;
    }
}

extern "C" size_t lb2_nn_table_bytes(void) { return (size_t)NNT_SLOTS * 12 + 16; }

extern "C" int lb2_nn_table_build(void* handle, void* stream, const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, void* table) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && k_coords && table && nk_cap > 0, "nn_table_build");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* tk = (unsigned long long*)table;
    int* tr = (int*)(tk + NNT_SLOTS);
    if (cudaMemsetAsync(tk, 0xFF, (size_t)NNT_SLOTS * 8, s) != cudaSuccess || cudaMemsetAsync(tr, 0x7F, (size_t)NNT_SLOTS * 4, s) != cudaSuccess)
        return lb2_fail(h, LB2_ERR_CUDA, "nn_table memset%s", "");
    k_nn_table_build<<<cdiv(nk_cap, 256), 256, 0, s>>>((const int4*)k_coords, d_nk, nk_cap, tk, tr, tr + NNT_SLOTS);
    LB2_POST_LAUNCH(h, "k_nn_table_build");
    return LB2_OK;
}

extern "C" int lb2_nn_match_table(void* handle, void* stream, const int32_t* q_coords, const int32_t* d_nq, int32_t nq_cap,
                                  const int32_t* k_coords, const int32_t* d_nk, int32_t nk_cap, const void* table,
                                  int32_t key_stride, int32_t max_ring, int32_t* idx) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && q_coords && k_coords && idx && table && nq_cap > 0 && nk_cap > 0, "nn_match_table");
    LB2_REQUIRE(h, key_stride > 0 && key_stride % 2 == 0 && max_ring >= 0 && max_ring <= 16, "nn_match_table stride/ring");
    {
        cudaError_t e = lb2_configure_smem(h, LB2_K_NN_TABLE, k_nn_match_table, NNT_SLOTS * 12);
        if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "k_nn_match_table smem attribute: %s", cudaGetErrorString(e));
    }
    const unsigned long long* tk = (const unsigned long long*)table;
    const int* tr = (const int*)(tk + NNT_SLOTS);
    const unsigned grid = std::min<unsigned>(h->num_sms, cdiv(nq_cap, NNT_THREADS));
    k_nn_match_table<<<grid, NNT_THREADS, NNT_SLOTS * 12, (cudaStream_t)stream>>>((const int4*)q_coords, d_nq, nq_cap, (const int4*)k_coords, d_nk, nk_cap,
                                                                                  tk, tr, key_stride, max_ring, idx);
    LB2_POST_LAUNCH(h, "k_nn_match_table");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// linear: y = act(x W^T + b + addend)
// ---------------------------------------------------------------------------------------------------
#define LIN_BM 64
#define LIN_BN 64
#define LIN_BK 16

__device__ __forceinline__ float lb2_act(float v, int act) {
    if (act == 1) return v > 0.f ? v : 0.1f * v;
    if (act == 2) return tanhf(v);
    return v;
}

__global__ void __launch_bounds__(256) k_linear(const float* __restrict__ x, long long ldx, const float* __restrict__ w,
                                                const float* __restrict__ b, const float* __restrict__ addend, long long ld_add,
                                                int m_cap, const int* __restrict__ d_m, int n_in, int n_out, int act,
                                                float* __restrict__ y, long long ldy,
                                                const float* __restrict__ prebias, int pre_act) {
    __shared__ float As[LIN_BK][LIN_BM + 4];
    __shared__ float Bs[LIN_BK][LIN_BN + 4];
    const int M = d_m ? min(*d_m, m_cap) : m_cap;
    const int m0 = blockIdx.x * LIN_BM, n0 = blockIdx.y * LIN_BN;
    if (m0 >= M) return;
    const int t = threadIdx.x, ty = t >> 4, tx = t & 15;
    const int lr = t >> 2, lc = (t & 3) * 4;       // loader: row lr (of 64), k offset lc..lc+3
    float acc[4][4] = {};
    for (int k0 = 0; k0 < n_in; k0 += LIN_BK) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + lc + j;
            const int row = m0 + lr, col = n0 + lr;
            float xv = 0.f;
            if (row < M && k < n_in) {
                xv = __ldg(x + (long long)row * ldx + k);
                if (prebias) xv = lb2_act(xv + __ldg(prebias + k), pre_act);
            }
            As[lc + j][lr] = xv;
            Bs[lc + j][lr] = (col < n_out && k < n_in) ? __ldg(w + (long long)col * n_in + k) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < LIN_BK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 bb = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = m0 + ty * 4 + i;
        if (row >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = n0 + tx * 4 + j;
            if (col >= n_out) continue;
            float v = acc[i][j];
            if (b) v += __ldg(b + col);
            if (addend) v += __ldg(addend + (long long)row * ld_add + col);
            y[(long long)row * ldy + col] = lb2_act(v, act);
        }
    }
}

extern "C" int lb2_linear(void* handle, void* stream, const float* x, int64_t ldx, const float* w, const float* b,
                          const float* addend, int64_t ld_addend, int32_t m_cap, const int32_t* d_m,
                          int32_t n_in, int32_t n_out, int32_t act, float* y, int64_t ldy,
                          const float* prebias, int32_t pre_act) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && x && w && y && m_cap > 0 && n_in > 0 && n_out > 0 && ldx >= n_in && ldy >= n_out, "linear");
    LB2_REQUIRE(h, !addend || ld_addend >= n_out, "linear: ld_addend < n_out");
    dim3 grid(cdiv(m_cap, LIN_BM), cdiv(n_out, LIN_BN));
    k_linear<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, w, b, addend, ld_addend, m_cap, d_m, n_in, n_out, act, y, ldy, prebias, pre_act);
    LB2_POST_LAUNCH(h, "k_linear");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// head MLP of the U-Nets (minkunet.py:376-380, :585-588): y = out_act(W1 . leaky_relu(W0 . x + b0, 0.1) + b1) in one pass over the rows,
// the hidden vector never leaves the registers.  Four lanes share a row (each n_in / 4 input channels, coalesced 64-byte pieces),
// the weights sit in shared memory; blockIdx.y = guidance pass.  Memory-bound: one read of x (rows x n_in fp32).
// ---------------------------------------------------------------------------------------------------
template <int NOUT_MAX>
__global__ void __launch_bounds__(256) k_head_mlp(const float* __restrict__ x, long long ldx, long long x_pass_stride,
                                                  const float* __restrict__ w0, const float* __restrict__ b0,
                                                  const float* __restrict__ w1, const float* __restrict__ b1, int m_cap,
                                                  const int* __restrict__ d_m, int n_in, int n_hid, int n_out, int out_act,
                                                  float* __restrict__ y, long long ldy, long long y_pass_stride) {
    extern __shared__ float hm_s[];
    float* w0s = hm_s;                                   // [n_hid][n_in]
    float* b0s = w0s + n_hid * n_in;                     // [n_hid]
    float* w1s = b0s + n_hid;                            // [n_out][n_hid]
    float* b1s = w1s + n_out * n_hid;                    // [n_out]
    for (int i = threadIdx.x; i < n_hid * n_in; i += blockDim.x) w0s[i] = __ldg(w0 + i);
    for (int i = threadIdx.x; i < n_hid; i += blockDim.x) b0s[i] = b0 ? __ldg(b0 + i) : 0.f;
    for (int i = threadIdx.x; i < n_out * n_hid; i += blockDim.x) w1s[i] = __ldg(w1 + i);
    for (int i = threadIdx.x; i < n_out; i += blockDim.x) b1s[i] = b1 ? __ldg(b1 + i) : 0.f;
    __syncthreads();
    const int M = d_m ? min(*d_m, m_cap) : m_cap;
    x += (long long)blockIdx.y * x_pass_stride;
    y += (long long)blockIdx.y * y_pass_stride;
    const int q = threadIdx.x & 3, nk = n_in >> 4;       // this lane's 16-byte piece of every 64 input bytes; pieces per row (<= 8)
    for (long long row = (long long)blockIdx.x * (blockDim.x >> 2) + (threadIdx.x >> 2); row < (long long)((M + 7) & ~7);
         row += (long long)gridDim.x * (blockDim.x >> 2)) {                      // whole groups of 8 rows per warp: the shuffles need every lane
        const bool live = row < M;
        float4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
            v[k] = (live && k < nk) ? __ldg(reinterpret_cast<const float4*>(x + row * ldx + k * 16 + q * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        float o[NOUT_MAX];
#pragma unroll
        for (int c = 0; c < NOUT_MAX; ++c) o[c] = 0.f;
        for (int j = 0; j < n_hid; ++j) {
            const float* wr = w0s + j * n_in + q * 4;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (k < nk) {
                    const float4 w = *reinterpret_cast<const float4*>(wr + k * 16);
                    s = fmaf(v[k].x, w.x, s); s = fmaf(v[k].y, w.y, s); s = fmaf(v[k].z, w.z, s); s = fmaf(v[k].w, w.w, s);
                }
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += b0s[j];
            s = s > 0.f ? s : 0.1f * s;                  // LeakyReLU(0.1)
#pragma unroll
            for (int c = 0; c < NOUT_MAX; ++c)
                if (c < n_out) o[c] = fmaf(w1s[c * n_hid + j], s, o[c]);
        }
        if (live && q == 0) {
#pragma unroll
            for (int c = 0; c < NOUT_MAX; ++c)
                if (c < n_out) y[row * ldy + c] = lb2_act(o[c] + b1s[c], out_act);
        }
    }
}

extern "C" int lb2_head_mlp(void* handle, void* stream, const float* x, int64_t ldx, int64_t x_pass_stride, const float* w0, const float* b0,
                            const float* w1, const float* b1, int32_t m_cap, const int32_t* d_m, int32_t n_in, int32_t n_hid,
                            int32_t n_out, int32_t out_act, int32_t npass, float* y, int64_t ldy, int64_t y_pass_stride) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && x && w0 && w1 && y && m_cap > 0 && npass >= 1 && npass <= 2, "head_mlp");
    LB2_REQUIRE(h, n_in >= 16 && n_in <= 128 && n_in % 16 == 0 && n_hid >= 1 && n_hid <= 64 && n_out >= 1 && n_out <= 24 && ldx >= n_in &&
                   ldx % 4 == 0 && ldy >= n_out, "head_mlp shape");
    // every row is read with float4 loads: the base of each pass must be 16-byte aligned
    LB2_REQUIRE(h, (uintptr_t)x % 16 == 0 && (npass == 1 || x_pass_stride % 4 == 0), "head_mlp: x or x_pass_stride not 16-byte aligned");
    const size_t smem = ((size_t)n_hid * n_in + n_hid + (size_t)n_out * n_hid + n_out) * sizeof(float);
    const dim3 grid((unsigned)std::min<long long>(cdiv(m_cap, 64), (long long)h->num_sms * 8), (unsigned)npass);
    if (n_out <= 4)
        k_head_mlp<4><<<grid, 256, smem, (cudaStream_t)stream>>>(x, ldx, x_pass_stride, w0, b0, w1, b1, m_cap, d_m, n_in, n_hid, n_out, out_act, y, ldy, y_pass_stride);
    else
        k_head_mlp<24><<<grid, 256, smem, (cudaStream_t)stream>>>(x, ldx, x_pass_stride, w0, b0, w1, b1, m_cap, d_m, n_in, n_hid, n_out, out_act, y, ldy, y_pass_stride);
    LB2_POST_LAUNCH(h, "k_head_mlp");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// gate multiply / row gather
// ---------------------------------------------------------------------------------------------------
__global__ void k_gate_mul(const float* __restrict__ x, const float* __restrict__ table, const int* __restrict__ idx,
                           const int* __restrict__ d_m, int m_cap, int c, float* __restrict__ out, __half* __restrict__ out_h) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int M = d_m ? min(*d_m, m_cap) : m_cap;
    if (t >= (long long)M * c) return;
    const int r = (int)(t / c), j = (int)(t % c);
    const int g = idx ? __ldg(idx + r) : 0;
    const float y = x[t] * __ldg(table + (long long)g * c + j);
    if (out) out[t] = y;
    if (out_h) {
        __half hi, lo;
        tc::split1(y, hi, lo);
        out_h[(long long)r * 2 * c + j] = hi;
        out_h[(long long)r * 2 * c + c + j] = lo;
    }
}

extern "C" int lb2_gate_mul(void* handle, void* stream, const float* x, const float* table, const int32_t* idx,
                            const int32_t* d_m, int32_t m_cap, int32_t c, float* out, void* out_h) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && x && table && (out || out_h) && m_cap > 0 && c > 0, "gate_mul");
    k_gate_mul<<<cdiv((long long)m_cap * c, 256), 256, 0, (cudaStream_t)stream>>>(x, table, idx, d_m, m_cap, c, out, (__half*)out_h);
    LB2_POST_LAUNCH(h, "k_gate_mul");
    return LB2_OK;
}

__global__ void k_gather_rows(const float* __restrict__ src, const int* __restrict__ idx, int n, int c, float* __restrict__ out) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * c) return;
    const int r = (int)(t / c), j = (int)(t % c);
    out[t] = __ldg(src + (long long)__ldg(idx + r) * c + j);
}

extern "C" int lb2_gather_rows(void* handle, void* stream, const float* src, const int32_t* idx, int32_t n, int32_t c, float* out) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && src && idx && out && n > 0 && c > 0, "gather_rows");
    k_gather_rows<<<cdiv((long long)n * c, 256), 256, 0, (cudaStream_t)stream>>>(src, idx, n, c, out);
    LB2_POST_LAUNCH(h, "k_gather_rows");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// guidance + DPM-Solver++(2M) SDE step + next-step features/coordinates, one thread per scalar.
// Arithmetic order and precisions follow the torch expressions of the reference exactly (no FMA
// contraction: explicit _rn intrinsics) so that, given identical eps, x_next and the coordinates
// are bit-identical to the fp64 torch evaluation.
// ---------------------------------------------------------------------------------------------------
__global__ void k_guidance_dpm(const float* __restrict__ eps_c, const float* __restrict__ eps_u, const int* __restrict__ inverse,
                               const float* __restrict__ x_t, const double* __restrict__ x_init, const float* __restrict__ noise,
                               double* __restrict__ x0_state, long long n_points, lb2_dpm_coef cf, float inv_res,
                               float* __restrict__ eps_out, float* __restrict__ x_next, float* __restrict__ coord_next,
                               const float* __restrict__ batch_col) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_points * 3) return;
    const long long pnt = t / 3;
    const int c = (int)(t - pnt * 3);
    const long long v = inverse ? (long long)__ldg(inverse + pnt) : pnt;
    const float ec = __ldg(eps_c + v * 3 + c), eu = __ldg(eps_u + v * 3 + c);
    // pipeline:153  x_uncond + w * (x_cond - x_uncond)   (fp32)
    const float eps = __fadd_rn(eu, __fmul_rn(cf.guidance_w, __fsub_rn(ec, eu)));
    if (eps_out) eps_out[t] = eps;
    // pipeline:162  input_noise = x_t.F - x_init   (fp32 - fp64 -> fp64)
    const double sample = __dsub_rn((double)x_t[t], x_init[t]);
    // diffusers convert_model_output: x0 = (sample - sigma_t * eps) / alpha_t   (sigma*eps in fp32)
    const double se = (double)__fmul_rn((float)cf.sigma_s, eps);
    const double x0 = __ddiv_rn(__dsub_rn(sample, se), cf.alpha_s);
    double prev = __dadd_rn(__dmul_rn(cf.c_sample, sample), __dmul_rn(cf.c_x0, x0));
    if (cf.second_order) {
        const double d1 = __dmul_rn(cf.inv_r0, __dsub_rn(x0, x0_state[t]));
        prev = __dadd_rn(prev, __dmul_rn(0.5 * cf.c_x0, d1));
    }
    // diffusers draws the SDE noise in the model output's dtype (fp32): sigma_t*sqrt(..) * noise is an fp32 product, promoted on the add
    prev = __dadd_rn(prev, (double)__fmul_rn((float)cf.c_noise, noise[t]));
    x0_state[t] = x0;
    // pipeline:163-164  x_t = x_init + prev ; batched_coordinates(dtype=float32)
    const float xn = __double2float_rn(__dadd_rn(x_init[t], prev));
    x_next[t] = xn;
    if (coord_next) {
        coord_next[pnt * 4 + 1 + c] = rintf(cf.div_mode == 0 ? __fdiv_rn(xn, cf.resolution) : __fmul_rn(xn, inv_res));
        if (c == 0) coord_next[pnt * 4] = batch_col ? batch_col[pnt] : 0.f;
    }
}

extern "C" int lb2_guidance_dpm_step(void* handle, void* stream, const float* eps_c, const float* eps_u,
                                     const int32_t* inverse, const float* x_t, const double* x_init,
                                     const float* noise, double* x0_state, int64_t n_points, lb2_dpm_coef coef,
                                     float* eps_out, float* x_next, float* coord_next, const float* batch_col) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && eps_c && eps_u && x_t && x_init && noise && x0_state && x_next && n_points > 0, "guidance_dpm_step");
    LB2_REQUIRE(h, coef.resolution > 0.f, "resolution");
    const float inv_res = 1.0f / coef.resolution;
    k_guidance_dpm<<<cdiv(n_points * 3, 256), 256, 0, (cudaStream_t)stream>>>(eps_c, eps_u, inverse, x_t, x_init, noise, x0_state,
                                                                              n_points, coef, inv_res, eps_out, x_next, coord_next, batch_col);
    LB2_POST_LAUNCH(h, "k_guidance_dpm");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// farthest point sampling: one CTA, running min squared distance in global (L2-resident), fp64
// ---------------------------------------------------------------------------------------------------
#define FPS_THREADS 1024

__global__ void __launch_bounds__(FPS_THREADS) k_fps(const double* __restrict__ pts, int n, int n_samples,
                                                      int* __restrict__ out_idx, double* __restrict__ dist) {
    __shared__ double s_val[FPS_THREADS / 32];
    __shared__ int s_idx[FPS_THREADS / 32];
    __shared__ int s_cur;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    for (int j = t; j < n; j += FPS_THREADS) dist[j] = DBL_MAX;
    if (t == 0) s_cur = 0;
    __syncthreads();
    for (int it = 0; it < n_samples; ++it) {
        const int cur = s_cur;
        if (t == 0) out_idx[it] = cur;
        const double cx = pts[3 * (long long)cur], cy = pts[3 * (long long)cur + 1], cz = pts[3 * (long long)cur + 2];
        double bv = -1.0; int bi = 0x7fffffff;
        for (int j = t; j < n; j += FPS_THREADS) {
            const double dx = pts[3 * (long long)j] - cx, dy = pts[3 * (long long)j + 1] - cy, dz = pts[3 * (long long)j + 2] - cz;
            // Eigen squaredNorm: x*x + y*y + z*z, left to right, no contraction
            double d = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            d = fmin(dist[j], d);
            dist[j] = d;
            if (d > bv) { bv = d; bi = j; }          // ascending j within a thread => first index kept
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        __syncthreads();          // previous iteration's readers of s_cur / s_val are done
        if (lane == 0) { s_val[w] = bv; s_idx[w] = bi; }
        __syncthreads();
        if (w == 0) {
            bv = s_val[lane]; bi = s_idx[lane];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) s_cur = bi;
        }
        __syncthreads();
    }
}

// ---- multi-CTA variant: every SM owns a slice of the points in REGISTERS; one grid barrier per sample ------------
struct FpsBest { double d; int idx; int pad; };
#define FPS_PPT 4

__global__ void __launch_bounds__(FPS_THREADS, 1) k_fps_coop(const double* __restrict__ pts, int n, int n_samples, int* __restrict__ out_idx,
                                                              FpsBest* blk_best /* [2][gridDim.x] */, unsigned* counter) {
    __shared__ double s_val[FPS_THREADS / 32];
    __shared__ int s_idx[FPS_THREADS / 32];
    __shared__ int s_cur;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int G = gridDim.x * FPS_THREADS, gtid = blockIdx.x * FPS_THREADS + t;
    double px[FPS_PPT], py[FPS_PPT], pz[FPS_PPT], dist[FPS_PPT];
#pragma unroll
    for (int q = 0; q < FPS_PPT; ++q) {
        const long long j = (long long)gtid + (long long)q * G;
        const bool ok = j < n;
        px[q] = ok ? pts[3 * j] : 0.0; py[q] = ok ? pts[3 * j + 1] : 0.0; pz[q] = ok ? pts[3 * j + 2] : 0.0;
        dist[q] = ok ? DBL_MAX : -1.0;                 // -1: slot unused, can never win
    }
    int cur = 0;
    for (int it = 0; it < n_samples; ++it) {
        if (gtid == 0) out_idx[it] = cur;
        const double cx = __ldg(pts + 3 * (long long)cur), cy = __ldg(pts + 3 * (long long)cur + 1), cz = __ldg(pts + 3 * (long long)cur + 2);
        double bv = -1.0; int bi = 0x7fffffff;
#pragma unroll
        for (int q = 0; q < FPS_PPT; ++q) {
            if (dist[q] >= 0.0) {
                const double dx = px[q] - cx, dy = py[q] - cy, dz = pz[q] - cz;
                const double d = fmin(dist[q], __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
                dist[q] = d;
                if (d > bv) { bv = d; bi = gtid + q * G; }       // ascending index per thread
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { s_val[w] = bv; s_idx[w] = bi; }
        __syncthreads();
        FpsBest* slot = blk_best + (size_t)(it & 1) * gridDim.x;
        if (w == 0) {
            bv = s_val[lane]; bi = s_idx[lane];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) {
                slot[blockIdx.x].d = bv; slot[blockIdx.x].idx = bi;
                __threadfence();
                atomicAdd(counter, 1u);
                const unsigned target = (unsigned)(it + 1) * gridDim.x;
                while (*(volatile unsigned*)counter < target) { }      // grid barrier (all CTAs co-resident: cooperative launch)
                __threadfence();
            }
            __syncwarp();
            bv = -1.0; bi = 0x7fffffff;
            for (int b = lane; b < (int)gridDim.x; b += 32) {
                const double ov = __ldcg(&slot[b].d);
                const int oi = __ldcg(&slot[b].idx);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) s_cur = bi;
        }
        __syncthreads();
        cur = s_cur;
    }
}

extern "C" int lb2_farthest_point_sample(void* handle, void* stream, const double* pts, int32_t n, int32_t n_samples,
                                         int32_t* out_idx, double* dist_scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && pts && out_idx && dist_scratch && n > 0 && n_samples > 0 && n_samples <= n, "fps");
    cudaStream_t s = (cudaStream_t)stream;
    const long long coop_cap = (long long)h->num_sms * FPS_THREADS * FPS_PPT;
    const size_t need = 2 * (size_t)h->num_sms * sizeof(FpsBest) + 64;
    if (n >= 8192 && n <= coop_cap && (size_t)n * sizeof(double) >= need && (long long)n_samples * h->num_sms < 0x7fffffffLL) {
        // cooperative multi-CTA kernel; scratch: [counter | pad][2][num_sms] FpsBest, carved from dist_scratch
        unsigned* counter = (unsigned*)dist_scratch;
        FpsBest* best = (FpsBest*)((char*)dist_scratch + 64);
        if (cudaMemsetAsync(counter, 0, 64, s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "fps memset%s", "");
        void* args[] = {(void*)&pts, (void*)&n, (void*)&n_samples, (void*)&out_idx, (void*)&best, (void*)&counter};
        cudaError_t e = cudaLaunchCooperativeKernel((const void*)k_fps_coop, dim3(h->num_sms), dim3(FPS_THREADS), args, 0, s);
        if (e == cudaSuccess) { h->launches++; return LB2_OK; }
        (void)cudaGetLastError();                      // cooperative launch unavailable: fall through to the single-CTA kernel
    }
    k_fps<<<1, FPS_THREADS, 0, s>>>(pts, n, n_samples, out_idx, dist_scratch);
    LB2_POST_LAUNCH(h, "k_fps");
    return LB2_OK;
}

// ---- batched: one thread-block cluster per scan, the scan on-chip -----------------------------------------------
// CTA r of a cluster owns the points [r*slice, (r+1)*slice) of its scan: coordinates in shared memory (SoA fp64), running
// distances in registers (FPS_CL_PPT per thread).  Each sample: thread argmax, warp and CTA reduction, the CTA's best goes
// into its own shared slot, one barrier.cluster, and every warp reduces the cluster's slots through distributed shared
// memory.  The slots are double-buffered by sample parity: a CTA writes slot[p] of sample it+2 only after the barrier of
// sample it+1, which every CTA passes after it has read slot[p] of sample it.  Same arithmetic and tie rule as k_fps_coop.
#define FPS_CL_PPT 9
#define FPS_CL_SLICE (FPS_THREADS * FPS_CL_PPT)          // 9216 points, 216 KB of coordinates per CTA

__global__ void __launch_bounds__(FPS_THREADS, 1) k_fps_cluster(const double* __restrict__ pts, const int64_t* __restrict__ offsets,
                                                                 int slice, int n_samples, int* __restrict__ out_idx) {
    namespace cg = cooperative_groups;
    extern __shared__ double fc_smem[];
    __shared__ double s_val[FPS_THREADS / 32];
    __shared__ int s_idx[FPS_THREADS / 32];
    __shared__ FpsBest s_slot[2];
    cg::cluster_group cl = cg::this_cluster();
    const int cs = (int)cl.num_blocks(), rank = (int)cl.block_rank();
    const int scan = blockIdx.x / cs;
    const long long off = offsets[scan];
    const int n = (int)(offsets[scan + 1] - off);
    const double* p = pts + 3 * off;
    double* sx = fc_smem;
    double* sy = sx + slice;
    double* sz = sy + slice;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int base = rank * slice, cnt = max(0, min(slice, n - base));
    for (int j = t; j < cnt; j += FPS_THREADS) {
        sx[j] = p[3 * (long long)(base + j)]; sy[j] = p[3 * (long long)(base + j) + 1]; sz[j] = p[3 * (long long)(base + j) + 2];
    }
    double dist[FPS_CL_PPT];
#pragma unroll
    for (int q = 0; q < FPS_CL_PPT; ++q) dist[q] = (t + q * FPS_THREADS < cnt) ? DBL_MAX : -1.0;   // -1: slot unused, can never win
    __syncthreads();
    int cur = 0;
    for (int it = 0; it < n_samples; ++it) {
        if (rank == 0 && t == 0) out_idx[(long long)scan * n_samples + it] = cur;
        // the centre from global memory (L2): carrying it in the cluster slots instead measured 1.8x slower (DESIGN.md §3)
        const double cx = __ldg(p + 3 * (long long)cur), cy = __ldg(p + 3 * (long long)cur + 1), cz = __ldg(p + 3 * (long long)cur + 2);
        double bv = -1.0; int bi = 0x7fffffff;
#pragma unroll
        for (int q = 0; q < FPS_CL_PPT; ++q) {
            if (dist[q] >= 0.0) {
                const int j = t + q * FPS_THREADS;
                const double dx = sx[j] - cx, dy = sy[j] - cy, dz = sz[j] - cz;
                const double d = fmin(dist[q], __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
                dist[q] = d;
                if (d > bv) { bv = d; bi = base + j; }                 // ascending index per thread
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { s_val[w] = bv; s_idx[w] = bi; }
        __syncthreads();
        if (w == 0) {
            bv = s_val[lane]; bi = s_idx[lane];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) { s_slot[it & 1].d = bv; s_slot[it & 1].idx = bi; }
        }
        cl.sync();                                                     // barrier.cluster arrive.release / wait.acquire
        bv = -1.0; bi = 0x7fffffff;
        if (lane < cs) {
            const FpsBest* r = cl.map_shared_rank(&s_slot[it & 1], lane);
            bv = r->d; bi = r->idx;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        cur = bi;
    }
    cl.sync();                                                         // no CTA exits while another may still read its slots
}

// cluster size for the batched kernel: 16 (non-portable) where the device can co-schedule it, else 8; 0 if neither
static int fps_cluster_size(Lb2Handle* h) {
    static const size_t smem = (size_t)3 * FPS_CL_SLICE * sizeof(double);
    if (lb2_configure_smem(h, LB2_K_FPS_CLUSTER, k_fps_cluster, (int)smem) != cudaSuccess) return 0;
    if (cudaFuncSetAttribute(k_fps_cluster, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
    for (int cs = 16; cs >= 8; cs /= 2) {
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3(cs); cfg.blockDim = dim3(FPS_THREADS); cfg.dynamicSmemBytes = smem; cfg.attrs = attr; cfg.numAttrs = 1;
        int nclusters = 0;
        if (cudaOccupancyMaxActiveClusters(&nclusters, k_fps_cluster, &cfg) == cudaSuccess && nclusters > 0) return cs;
        (void)cudaGetLastError();
    }
    return 0;
}

extern "C" int64_t lb2_fps_batched_capacity(void* handle) {
    Lb2Handle* h = (Lb2Handle*)handle;
    if (!h) return 0;
    return (int64_t)fps_cluster_size(h) * FPS_CL_SLICE;
}

extern "C" int lb2_farthest_point_sample_batched(void* handle, void* stream, const double* pts, const int64_t* d_offsets, int32_t n_scans,
                                                 int32_t max_n, int32_t n_samples, int32_t* out_idx) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h && pts && d_offsets && out_idx && n_scans > 0 && max_n > 0 && n_samples > 0 && n_samples <= max_n, "fps_batched");
    const int cs = fps_cluster_size(h);
    if (cs == 0) return lb2_fail(h, LB2_ERR_CUDA, "fps_batched: the device cannot run an 8-CTA cluster with %s of shared memory", "216 KB");
    LB2_REQUIRE(h, (long long)max_n <= (long long)cs * FPS_CL_SLICE, "fps_batched: a scan exceeds lb2_fps_batched_capacity()");
    LB2_REQUIRE(h, (long long)n_scans * cs <= 0x7fffffffLL, "fps_batched: too many scans");
    const int slice = (max_n + cs - 1) / cs;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)(n_scans * cs)); cfg.blockDim = dim3(FPS_THREADS);
    cfg.dynamicSmemBytes = (size_t)3 * slice * sizeof(double); cfg.stream = (cudaStream_t)stream; cfg.attrs = attr; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, k_fps_cluster, pts, d_offsets, slice, (int)n_samples, (int*)out_idx);
    if (e != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "k_fps_cluster: %s", cudaGetErrorString(e));
    LB2_POST_LAUNCH(h, "k_fps_cluster");
    return LB2_OK;
}
