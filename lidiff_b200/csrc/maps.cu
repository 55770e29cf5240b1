// Ground-truth map building — stands behind lidiff/map_from_scans.py:63-96 (filter, transform and re-de-duplicate the whole map after every
// scan).  A map point is never evicted by a later scan, so the map equals one pass of global first-occurrence de-duplication over the
// concatenation of all filtered, transformed scans; it is built here in streaming form: one persistent open-addressing table of voxel keys,
// each scan touches only its own points and appends its new voxels in first-occurrence order.  O(points read) instead of O(scans x map).
// Integer atomics only (key CAS, claim atomicMin), output order fixed by point order: deterministic.
#include "common.cuh"
#include <limits.h>

#define MAP_THREADS  512
#define MAP_ITEMS    4
#define MAP_TILE     (MAP_THREADS * MAP_ITEMS)

struct MapScratch {        // carved out of the caller's scratch buffer
    int* slot_of;          // [n_cap] table slot claimed by point i, -1 = dropped (filtered or voxel already in the map)
    int* rank;             // [n_cap] block-local rank of a winner, -1 = not a winner
    int* bsum;             // [MAP_TILE] block totals -> block offsets
};

static size_t map_align(int64_t n) { return ((size_t)n * sizeof(int) + 255) / 256 * 256; }

extern "C" size_t lb2_map_scan_scratch_bytes(int32_t n_cap) {
    return 2 * map_align(n_cap > 0 ? n_cap : 1) + MAP_TILE * sizeof(int) + 256;
}

static MapScratch map_carve(void* scratch, int32_t n_cap) {
    size_t a = map_align(n_cap > 0 ? n_cap : 1);
    char* p = (char*)scratch;
    MapScratch s;
    s.slot_of = (int*)p; s.rank = (int*)(p + a); s.bsum = (int*)(p + 2 * a);
    return s;
}

// Filter, transform and key of point i, in the arithmetic order of the header (no FMA contraction: explicit _rn intrinsics).
// Returns 0 = filtered out, 1 = kept (w, key valid), 2 = kept but its voxel index is outside the key range.
__device__ __forceinline__ int map_point(const float4* __restrict__ pts, const unsigned* __restrict__ labels, int i, const lb2_pose& P,
                                         float vs, float inv_vs, int div_mode, float3& w, unsigned long long& key) {
    if (labels) {
        unsigned l = __ldg(labels + i) & 0xFFFFu;
        if (!(l > 1u && l < 252u)) return 0;
    }
    float4 p = __ldg(pts + i);
    float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)), __fmul_rn(p.z, p.z)), __fmul_rn(p.w, p.w));
    if (!(__fsqrt_rn(s) > 3.5f)) return 0;
    float c[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        c[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.m[4 * r], p.x), __fmul_rn(P.m[4 * r + 1], p.y)), __fmul_rn(P.m[4 * r + 2], p.z)),
                         P.m[4 * r + 3]);
    w = make_float3(c[0], c[1], c[2]);
    key = 0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        float f = floorf(div_mode == 0 ? __fdiv_rn(c[r], vs) : __fmul_rn(c[r], inv_vs));
        if (!lb2_map_cell_ok(f)) return 2;
        key = lb2_map_key_push(key, (int)f);
    }
    return 1;
}

// a point whose voxel already has a map row is dropped; for a voxel without one, the lowest point index of this call wins
__global__ void __launch_bounds__(256) k_map_insert(const float4* __restrict__ pts, const unsigned* __restrict__ labels, int n, lb2_pose P,
                                                    float vs, float inv_vs, int div_mode, unsigned long long* keys, int* vals, int cap,
                                                    int* __restrict__ slot_of, int* __restrict__ d_out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float3 w;
    unsigned long long key;
    int st = map_point(pts, labels, i, P, vs, inv_vs, div_mode, w, key);
    int slot = -1;
    if (st == 2) atomicOr(d_out + 1, 1);
    if (st == 1) {
        unsigned s = lb2_key_insert(keys, (unsigned)cap - 1u, key);
        // rows are written only by k_map_emit of an earlier call; a slot without a row was created in this call
        if (vals[cap + s] < 0) {
            atomicMin(vals + s, i);
            slot = (int)s;
        }
    }
    slot_of[i] = slot;
}

// block-level exclusive scan of the "wins its slot" flags
__global__ void __launch_bounds__(MAP_THREADS) k_map_scan_local(const int* __restrict__ slot_of, const int* __restrict__ vals, int n,
                                                                int* __restrict__ rank, int* __restrict__ bsum) {
    __shared__ int warp_tot[MAP_THREADS / 32];
    int base = blockIdx.x * MAP_TILE + threadIdx.x * MAP_ITEMS;
    int f[MAP_ITEMS], tsum = 0;
#pragma unroll
    for (int j = 0; j < MAP_ITEMS; ++j) {
        int i = base + j, s = (i < n) ? slot_of[i] : -1;
        f[j] = (s >= 0) && (vals[s] == i);
        tsum += f[j];
    }
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int incl = tsum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    if (w == 0) {
        int v = (lane < MAP_THREADS / 32) ? warp_tot[lane] : 0, inc2 = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc2, d); if (lane >= d) inc2 += u; }
        if (lane < MAP_THREADS / 32) warp_tot[lane] = inc2 - v;
        if (lane == MAP_THREADS / 32 - 1) bsum[blockIdx.x] = inc2;
    }
    __syncthreads();
    int excl = warp_tot[w] + incl - tsum;
#pragma unroll
    for (int j = 0; j < MAP_ITEMS; ++j) {
        int i = base + j;
        if (i < n) rank[i] = f[j] ? excl : -1;
        excl += f[j];
    }
}

// single block: exclusive scan of up to MAP_TILE block totals; the grand total is the number of new rows
__global__ void __launch_bounds__(MAP_THREADS) k_map_scan_bsum(int* __restrict__ bsum, int nblocks, int* __restrict__ d_out) {
    __shared__ int warp_tot[MAP_THREADS / 32];
    int base = threadIdx.x * MAP_ITEMS;
    int v[MAP_ITEMS], tsum = 0;
#pragma unroll
    for (int j = 0; j < MAP_ITEMS; ++j) { v[j] = (base + j < nblocks) ? bsum[base + j] : 0; tsum += v[j]; }
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int incl = tsum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += u; }
    if (lane == 31) warp_tot[w] = incl;
    __syncthreads();
    if (w == 0) {
        int x = (lane < MAP_THREADS / 32) ? warp_tot[lane] : 0, inc2 = x;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc2, d); if (lane >= d) inc2 += u; }
        if (lane < MAP_THREADS / 32) warp_tot[lane] = inc2 - x;
        if (lane == MAP_THREADS / 32 - 1) d_out[0] = inc2;
    }
    __syncthreads();
    int excl = warp_tot[w] + incl - tsum;
#pragma unroll
    for (int j = 0; j < MAP_ITEMS; ++j) { if (base + j < nblocks) bsum[base + j] = excl; excl += v[j]; }
}

// winners take the next map rows in point order, publish the row in their slot and append their transformed point
__global__ void __launch_bounds__(256) k_map_emit(const float4* __restrict__ pts, const unsigned* __restrict__ labels, int n, lb2_pose P,
                                                  float vs, float inv_vs, int div_mode, const int* __restrict__ slot_of,
                                                  const int* __restrict__ rank, const int* __restrict__ bsum, int* __restrict__ vals, int cap,
                                                  int map_n, float* __restrict__ map) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int r = rank[i];
    if (r < 0) return;
    r += bsum[i / MAP_TILE] + map_n;
    float3 w;
    unsigned long long key;
    map_point(pts, labels, i, P, vs, inv_vs, div_mode, w, key);     // the same inline arithmetic as k_map_insert: the same bits
    vals[cap + slot_of[i]] = r;
    map[3 * (size_t)r] = w.x; map[3 * (size_t)r + 1] = w.y; map[3 * (size_t)r + 2] = w.z;
}

extern "C" int lb2_map_scan(void* handle, void* stream, const float* points, const uint32_t* labels, int32_t n, lb2_pose pose,
                            float voxel_size, int32_t div_mode, lb2_grid table, float* map, int32_t map_n, int32_t map_cap,
                            int32_t* d_out, void* scratch) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, d_out && table.keys && table.vals && map, "null buffer");
    LB2_REQUIRE(h, n >= 0 && n <= MAP_TILE * MAP_TILE, "n out of range (max 4M points per call)");
    LB2_REQUIRE(h, voxel_size > 0.f && (div_mode == 0 || div_mode == 1), "voxel_size / div_mode");
    LB2_REQUIRE(h, table.cap_table >= 2 && (table.cap_table & (table.cap_table - 1)) == 0, "cap_table must be a power of two");
    LB2_REQUIRE(h, map_n >= 0 && (int64_t)table.cap_table >= 2 * ((int64_t)map_n + n), "cap_table must be >= 2 * (map_n + n)");
    LB2_REQUIRE(h, (int64_t)map_cap >= (int64_t)map_n + n, "map_cap must be >= map_n + n");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(d_out, 0, 2 * sizeof(int32_t), s) != cudaSuccess) return lb2_fail(h, LB2_ERR_CUDA, "%s", "cudaMemsetAsync");
    if (n == 0) return LB2_OK;
    LB2_REQUIRE(h, points && scratch, "null buffer");
    MapScratch sc = map_carve(scratch, n);
    float inv = 1.0f / voxel_size;       // fp32 reciprocal, as PyTorch's CUDA scalar-divide does
    int nblk = (int)cdiv(n, MAP_TILE);
    const float4* p4 = (const float4*)points;
    const unsigned* lab = (const unsigned*)labels;
    unsigned long long* keys = (unsigned long long*)table.keys;
    k_map_insert<<<cdiv(n, 256), 256, 0, s>>>(p4, lab, n, pose, voxel_size, inv, div_mode, keys, table.vals, table.cap_table,
                                              sc.slot_of, d_out);
    LB2_POST_LAUNCH(h, "k_map_insert");
    k_map_scan_local<<<nblk, MAP_THREADS, 0, s>>>(sc.slot_of, table.vals, n, sc.rank, sc.bsum);
    LB2_POST_LAUNCH(h, "k_map_scan_local");
    k_map_scan_bsum<<<1, MAP_THREADS, 0, s>>>(sc.bsum, nblk, d_out);
    LB2_POST_LAUNCH(h, "k_map_scan_bsum");
    k_map_emit<<<cdiv(n, 256), 256, 0, s>>>(p4, lab, n, pose, voxel_size, inv, div_mode, sc.slot_of, sc.rank, sc.bsum, table.vals,
                                            table.cap_table, map_n, map);
    LB2_POST_LAUNCH(h, "k_map_emit");
    return LB2_OK;
}

// ---------------------------------------------------------------------------------------------------
// growth: a fresh table at a larger capacity, filled with the (key, row) pairs of the old one
// ---------------------------------------------------------------------------------------------------
__global__ void k_map_clear(unsigned long long* keys, int* vals, int cap) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cap) { keys[i] = LB2_KEY_EMPTY; vals[i] = INT_MAX; vals[cap + i] = -1; }
}

__global__ void k_map_reinsert(const unsigned long long* __restrict__ old_keys, const int* __restrict__ old_vals, int old_cap,
                               unsigned long long* keys, int* vals, int cap) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= old_cap) return;
    unsigned long long key = old_keys[i];
    if (key == LB2_KEY_EMPTY) return;
    unsigned mask = (unsigned)cap - 1u, s = lb2_hash(key) & mask;
    while (atomicCAS(keys + s, (unsigned long long)LB2_KEY_EMPTY, key) != LB2_KEY_EMPTY) s = (s + 1) & mask;     // keys are distinct
    vals[cap + s] = old_vals[old_cap + i];
}

extern "C" int lb2_map_rehash(void* handle, void* stream, lb2_grid old_table, lb2_grid table) {
    Lb2Handle* h = (Lb2Handle*)handle;
    LB2_REQUIRE(h, h != nullptr, "handle");
    LB2_REQUIRE(h, table.keys && table.vals, "null buffer");
    LB2_REQUIRE(h, table.cap_table >= 2 && (table.cap_table & (table.cap_table - 1)) == 0, "cap_table must be a power of two");
    bool has_old = old_table.keys != nullptr && old_table.cap_table > 0;
    LB2_REQUIRE(h, !has_old || (old_table.vals && old_table.cap_table <= table.cap_table), "old table larger than the new one");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long* keys = (unsigned long long*)table.keys;
    k_map_clear<<<cdiv(table.cap_table, 256), 256, 0, s>>>(keys, table.vals, table.cap_table);
    LB2_POST_LAUNCH(h, "k_map_clear");
    if (has_old) {
        k_map_reinsert<<<cdiv(old_table.cap_table, 256), 256, 0, s>>>((const unsigned long long*)old_table.keys, old_table.vals,
                                                                      old_table.cap_table, keys, table.vals, table.cap_table);
        LB2_POST_LAUNCH(h, "k_map_reinsert");
    }
    return LB2_OK;
}
