// lbvh.cu -- GPU-built linear BVH (Morton keys + radix sort + Karras hierarchy + bottom-up refit).
//
// Replaces the driver-opaque acceleration structure the reference builds with
// vkCmdBuildAccelerationStructuresKHR (VulkanHelper/Source/Vulkan/BLASBuilderImpl.cpp:196-273, TLASImpl.cpp:100-190;
// one BLAS per mesh instance, PathTracer/PathTracer.cpp:449-502).  The two-level TLAS/BLAS is flattened into one
// world-space BVH2 (all shipped scenes are static), keeping (InstanceIndex, PrimitiveIndex) per triangle because
// the emissive-mesh NEE visibility test compares them (PathTracer/Shaders/ClosestHit.slang:171-176).
//
// Output layout (one contiguous allocation so small scenes are staged into shared memory with one TMA bulk copy):
//   [ BvhNode x max(N-1,1) | BvhTri x N ]   nodes: 64 B, both child boxes in the parent; tris: 48 B, Morton order.
#include "kernels.h"
#include "bvh_build_rules.cuh"
#include <vector>
#include <condition_variable>
#include <mutex>
#include <functional>
#include <thread>
#include <cstring>
#include <cstdlib>
#include <algorithm>
#include <cstdio>

namespace b200pt {

#ifndef LBVH_LEAF_MAX
#define LBVH_LEAF_MAX 4
#endif
#ifndef LBVH_SIZE_CLASS
#define LBVH_SIZE_CLASS 0
#endif
#ifndef LBVH_SPLIT_MAX
#define LBVH_SPLIT_MAX 16
#endif
#define LBVH_CHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

// world-space transform without FMA contraction: bit-identical to the CPU oracle's plain fp32 arithmetic
__device__ __forceinline__ float dot3_1_rn(float a, float b, float c, float d, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, x), __fmul_rn(b, y)), __fmul_rn(c, z)), __fmul_rn(d, 1.0f));
}
__device__ __forceinline__ float3 xf_point_rn(const float *m, float x, float y, float z) {
    return make_float3(dot3_1_rn(m[0], m[1], m[2], m[3], x, y, z), dot3_1_rn(m[4], m[5], m[6], m[7], x, y, z), dot3_1_rn(m[8], m[9], m[10], m[11], x, y, z));
}

__device__ __forceinline__ void atomic_min_f(float *addr, float v) {   // works for any sign via ordered ints
    v += 0.0f;                                                           // -0.0 -> +0.0: its bit pattern (INT_MIN) would win every signed atomicMin
    if (v >= 0.0f) atomicMin(reinterpret_cast<int *>(addr), __float_as_int(v));
    else atomicMax(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_f(float *addr, float v) {
    v += 0.0f;
    if (v >= 0.0f) atomicMax(reinterpret_cast<int *>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v));
}

// ---- 1. world triangles + scene bounds -------------------------------------------------------
__device__ __forceinline__ uint32_t instance_of(const DevInstance *__restrict__ inst, uint32_t n_inst, uint32_t gid) {
    uint32_t a = 0, b = n_inst - 1;                                      // last instance with tri_base <= gid
    while (a < b) { uint32_t mid = (a + b + 1) >> 1; if (inst[mid].tri_base <= gid) a = mid; else b = mid - 1; }
    return a;
}
// The 48-B record of global triangle gid (primitive prim of instance a) and its world box bb (lo xyz, hi xyz).  k_world_tris and the refit
// (k_refit_slots) both call this, so a refit slot holds exactly the record a fresh build of the moved scene would hold.
__device__ __forceinline__ BvhTri world_tri(const DevInstance &in, uint32_t a, uint32_t gid, uint32_t prim, const b200pt_vertex &A, const b200pt_vertex &B,
                                            const b200pt_vertex &C, float bb[6]) {
    const float3 v0 = xf_point_rn(in.o2w, A.Position[0], A.Position[1], A.Position[2]);
    const float3 v1 = xf_point_rn(in.o2w, B.Position[0], B.Position[1], B.Position[2]);
    const float3 v2 = xf_point_rn(in.o2w, C.Position[0], C.Position[1], C.Position[2]);
    BvhTri t;
    t.a = make_float4(v0.x, v0.y, v0.z, __uint_as_float(gid));
    t.b = make_float4(__fsub_rn(v1.x, v0.x), __fsub_rn(v1.y, v0.y), __fsub_rn(v1.z, v0.z), __uint_as_float(a));
    t.c = make_float4(__fsub_rn(v2.x, v0.x), __fsub_rn(v2.y, v0.y), __fsub_rn(v2.z, v0.z), __uint_as_float(prim));
    bb[0] = fminf(v0.x, fminf(v1.x, v2.x)); bb[3] = fmaxf(v0.x, fmaxf(v1.x, v2.x));
    bb[1] = fminf(v0.y, fminf(v1.y, v2.y)); bb[4] = fmaxf(v0.y, fmaxf(v1.y, v2.y));
    bb[2] = fminf(v0.z, fminf(v1.z, v2.z)); bb[5] = fmaxf(v0.z, fmaxf(v1.z, v2.z));
    return t;
}
// The shading record of triangle prim of instance a: object-space positions, normals and UVs (a transform never changes it, a vertex update
// does).  k_world_tris and the vertex-update refresh (k_refresh_shade) both call this.
__device__ __forceinline__ ShadeTri shade_tri(uint32_t a, uint32_t prim, uint32_t material, const b200pt_vertex &A, const b200pt_vertex &B, const b200pt_vertex &C) {
    ShadeTri sh;
    sh.r[0] = make_float4(A.Position[0], A.Position[1], A.Position[2], __uint_as_float(a));
    sh.r[1] = make_float4(B.Position[0], B.Position[1], B.Position[2], __uint_as_float(prim));
    sh.r[2] = make_float4(C.Position[0], C.Position[1], C.Position[2], __uint_as_float(material));
    sh.r[3] = make_float4(A.Normal[0], A.Normal[1], A.Normal[2], A.TexCoord[0]);
    sh.r[4] = make_float4(B.Normal[0], B.Normal[1], B.Normal[2], A.TexCoord[1]);
    sh.r[5] = make_float4(C.Normal[0], C.Normal[1], C.Normal[2], B.TexCoord[0]);
    sh.r[6] = make_float4(B.TexCoord[1], C.TexCoord[0], C.TexCoord[1], 0.0f);
    return sh;
}
__device__ __forceinline__ void reduce_bounds(float lo[3], float hi[3], float *bounds) {   // warp-reduce, then one atomic per warp (whole warps call it)
    for (int k = 0; k < 3; k++) {
        for (int o = 16; o > 0; o >>= 1) { lo[k] = fminf(lo[k], __shfl_down_sync(0xFFFFFFFFu, lo[k], o)); hi[k] = fmaxf(hi[k], __shfl_down_sync(0xFFFFFFFFu, hi[k], o)); }
        if ((threadIdx.x & 31) == 0) { atomic_min_f(&bounds[k], lo[k]); atomic_max_f(&bounds[3 + k], hi[k]); }
    }
}
__global__ void k_world_tris(const b200pt_vertex *__restrict__ verts, const uint32_t *__restrict__ indices, const DevMesh *__restrict__ meshes,
                             const DevInstance *__restrict__ inst, uint32_t n_inst, uint32_t n_tris,
                             BvhTri *__restrict__ tmp, ShadeTri *__restrict__ shade, float *__restrict__ cent, float *__restrict__ bounds /*6*/) {
    const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
    float lo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, hi[3] = { -3.0e38f, -3.0e38f, -3.0e38f };
    if (gid < n_tris) {
        const uint32_t a = instance_of(inst, n_inst, gid);
        const DevInstance &in = inst[a];
        const uint32_t prim = gid - in.tri_base;
        const DevMesh m = meshes[in.mesh];
        const uint32_t *ix = indices + m.ibase + (size_t)prim * 3;
        const b200pt_vertex &A = verts[m.vbase + ix[0]], &B = verts[m.vbase + ix[1]], &C = verts[m.vbase + ix[2]];
        float bb[6];
        tmp[gid] = world_tri(in, a, gid, prim, A, B, C, bb);
        shade[gid] = shade_tri(a, prim, in.material, A, B, C);
        for (int k = 0; k < 3; k++) { lo[k] = bb[k]; hi[k] = bb[3 + k]; }
        for (int k = 0; k < 6; k++) cent[(size_t)gid * 6 + k] = bb[k];  // per-triangle AABB (unsorted)
    }
    reduce_bounds(lo, hi, bounds);
}

// ---- 1b. early split clipping: fat boxes of thin diagonal triangles are cut into up to 8 references ------------------
// BreakfastRoom's chair legs are 86,880 slivers (aspect ratio 240 at p90) lying diagonally: every sliver's AABB is as big as
// the whole tube, so a ray near a leg tested ~170 triangles.  Each reference is the AABB of the
// triangle clipped to one slab of its longest axis; all references of a triangle point to the same BvhTri.
__global__ void k_split_count(const BvhTri *__restrict__ tmp, const float *__restrict__ aabb, const float *__restrict__ bounds, uint32_t n, uint32_t *__restrict__ ksplit) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *bb = aabb + (size_t)i * 6;
    float e[3] = { bb[3] - bb[0], bb[4] - bb[1], bb[5] - bb[2] };
    if (e[0] < e[1]) { float t = e[0]; e[0] = e[1]; e[1] = t; }
    if (e[1] < e[2]) { float t = e[1]; e[1] = e[2]; e[2] = t; }
    if (e[0] < e[1]) { float t = e[0]; e[0] = e[1]; e[1] = t; }
    const float4 b = tmp[i].b, c = tmp[i].c;
    const float cx = b.y * c.z - b.z * c.y, cy = b.z * c.x - b.x * c.z, cz = b.x * c.y - b.y * c.x;
    const float area2 = sqrtf(cx * cx + cy * cy + cz * cz);
    const float scene = fmaxf(bounds[3] - bounds[0], fmaxf(bounds[4] - bounds[1], bounds[5] - bounds[2]));
    uint32_t k = 1;
    const float ratio = (e[0] * e[1]) / fmaxf(area2, 1e-30f);
    if (ratio > 8.0f && e[0] > scene * (1.0f / 1024.0f)) k = (uint32_t)fminf(fmaxf(ceilf(sqrtf(ratio)), 2.0f), (float)LBVH_SPLIT_MAX);
    ksplit[i] = k;
}
__device__ __forceinline__ int clip_poly(const float3 *in, int n, int axis, float plane, bool keep_greater, float3 *out) {
    int m = 0;
    for (int a = 0; a < n; a++) {
        const float3 P = in[a], Q = in[(a + 1) % n];
        const float pa = axis == 0 ? P.x : (axis == 1 ? P.y : P.z), qa = axis == 0 ? Q.x : (axis == 1 ? Q.y : Q.z);
        const bool pin = keep_greater ? pa >= plane : pa <= plane, qin = keep_greater ? qa >= plane : qa <= plane;
        if (pin) out[m++] = P;
        if (pin != qin) { const float t = (plane - pa) / (qa - pa); out[m++] = make_float3(P.x + t * (Q.x - P.x), P.y + t * (Q.y - P.y), P.z + t * (Q.z - P.z)); }
    }
    return m;
}
// Reference box of slab j of k (k >= 2) of triangle t with world box bb: slabs cut the longest axis of bb into k equal parts, so the k slabs
// cover the triangle whatever order they are taken in.  k_make_refs and the refit (k_refit_slots) both call this.
__device__ __forceinline__ void slab_ref_box(const BvhTri &t, const float *bb, uint32_t j, uint32_t k, float *o) {
    const float ex = bb[3] - bb[0], ey = bb[4] - bb[1], ez = bb[5] - bb[2];
    const int axis = (ex >= ey && ex >= ez) ? 0 : (ey >= ez ? 1 : 2);
    const float lo = bb[axis], w = (bb[3 + axis] - bb[axis]) / (float)k;
    const float3 v0 = make_float3(t.a.x, t.a.y, t.a.z), v1 = make_float3(t.a.x + t.b.x, t.a.y + t.b.y, t.a.z + t.b.z), v2 = make_float3(t.a.x + t.c.x, t.a.y + t.c.y, t.a.z + t.c.z);
    const float s0 = lo + w * (float)j, s1 = (j + 1 == k) ? bb[3 + axis] : lo + w * (float)(j + 1);
    float3 p0[8], p1[8];                                                 // a triangle clipped by two planes has <= 5 vertices
    p0[0] = v0; p0[1] = v1; p0[2] = v2;
    int m = clip_poly(p0, 3, axis, s0, true, p1);
    m = clip_poly(p1, m, axis, s1, false, p0);
    float blo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, bhi[3] = { -3.0e38f, -3.0e38f, -3.0e38f };
    for (int a = 0; a < m; a++) {
        blo[0] = fminf(blo[0], p0[a].x); blo[1] = fminf(blo[1], p0[a].y); blo[2] = fminf(blo[2], p0[a].z);
        bhi[0] = fmaxf(bhi[0], p0[a].x); bhi[1] = fmaxf(bhi[1], p0[a].y); bhi[2] = fmaxf(bhi[2], p0[a].z);
    }
    for (int q = 0; q < 3; q++) {
        float l = bb[q], h = bb[3 + q];
        if (q == axis) { l = s0; h = s1; }
        if (m >= 1) {                                                    // clipped polygon bounds, padded, never beyond the triangle's own box
            const float pad = 1e-5f * fmaxf(fabsf(blo[q]), fabsf(bhi[q])) + 1e-6f * (bb[3 + q] - bb[q]) + 1e-30f;
            l = fmaxf(l, blo[q] - pad); h = fminf(h, bhi[q] + pad);
            if (l > h) { l = bb[q]; h = bb[3 + q]; if (q == axis) { l = s0; h = s1; } }
        }
        o[q] = l; o[3 + q] = h;
    }
}
__global__ void k_make_refs(const BvhTri *__restrict__ tmp, const float *__restrict__ aabb, const uint32_t *__restrict__ ksplit, const uint32_t *__restrict__ ref_off,
                            uint32_t n, float *__restrict__ ref_box, uint32_t *__restrict__ ref_tri) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *bb = aabb + (size_t)i * 6;
    const uint32_t k = ksplit[i], r0 = ref_off[i];
    if (k == 1) { for (int q = 0; q < 6; q++) ref_box[(size_t)r0 * 6 + q] = bb[q]; ref_tri[r0] = i; return; }
    const BvhTri t = tmp[i];
    for (uint32_t j = 0; j < k; j++) {
        slab_ref_box(t, bb, j, k, ref_box + (size_t)(r0 + j) * 6);
        ref_tri[r0 + j] = i;
    }
}

// ---- 2. Morton keys ---------------------------------------------------------------------------
// 60-bit Morton keys (20 bits per axis) + 2 size-class bits: with 10 bits per axis every finely tessellated object collapses into a handful of
// 1.2-cm cells of equal key and Karras falls back to index order there (measured on BreakfastRoom: up to 647 triangle
// tests for one camera ray)
__device__ __forceinline__ unsigned long long expand_bits21(unsigned long long x) {
    x &= 0x1fffffull;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}
__global__ void k_morton(const float *__restrict__ aabb, const float *__restrict__ bounds, uint32_t n, unsigned long long *keys, uint32_t *vals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *bb = aabb + (size_t)i * 6;
    unsigned long long q[3];
    float rel = 0.0f;                                                     // largest extent of the triangle relative to the scene
    for (int k = 0; k < 3; k++) {
        const float c = 0.5f * (bb[k] + bb[3 + k]);
        const float ext = bounds[3 + k] - bounds[k];
        float f = ext > 0.0f ? (c - bounds[k]) / ext : 0.0f;
        if (ext > 0.0f) rel = fmaxf(rel, (bb[3 + k] - bb[k]) / ext);
        f = fminf(fmaxf(f * 1048576.0f, 0.0f), 1048575.0f);
        q[k] = (unsigned long long)f;
    }
    // Size class in the top key bits: a wall-sized triangle sorted by its centroid alone inflates every ancestor box on its
    // root-to-leaf path (BreakfastRoom: p99 143 / max 324 node visits per camera ray).  Sorting by (size class, Morton code)
    // makes Karras split by size first, so large triangles live in their own small subtrees next to the root.
    const unsigned long long cls = !LBVH_SIZE_CLASS ? 0ull : (rel > 0.25f ? 3ull : (rel > 0.0625f ? 2ull : (rel > 0.015625f ? 1ull : 0ull)));
    keys[i] = (cls << 60) | (expand_bits21(q[0]) << 2) | (expand_bits21(q[1]) << 1) | expand_bits21(q[2]);
    vals[i] = i;
}

// ---- 3. stable LSD radix sort, 4-bit digits, 256-element tiles ----------------------------------
__global__ void __launch_bounds__(256) k_radix_hist(const unsigned long long *__restrict__ keys, uint32_t n, int shift, uint32_t *__restrict__ hist, uint32_t nblocks) {
    __shared__ uint32_t cnt[16];
    if (threadIdx.x < 16) cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) atomicAdd(&cnt[(uint32_t)(keys[i] >> shift) & 15u], 1u);
    __syncthreads();
    if (threadIdx.x < 16) hist[threadIdx.x * nblocks + blockIdx.x] = cnt[threadIdx.x];
}
__global__ void __launch_bounds__(1024) k_radix_scan(uint32_t *__restrict__ hist, uint32_t total) {   // exclusive scan, single block
    __shared__ uint32_t sm[1024];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < total; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < total ? hist[i] : 0u;
        sm[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            uint32_t t = threadIdx.x >= (unsigned)o ? sm[threadIdx.x - o] : 0u;
            __syncthreads();
            sm[threadIdx.x] += t;
            __syncthreads();
        }
        const uint32_t incl = sm[threadIdx.x];
        if (i < total) hist[i] = carry + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += incl;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) k_radix_scatter(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ vals, uint32_t n, int shift,
                                                        const uint32_t *__restrict__ hist, uint32_t nblocks, unsigned long long *__restrict__ keys_out, uint32_t *__restrict__ vals_out) {
    __shared__ uint32_t wcnt[8][17];
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const bool act = i < n;
    const unsigned long long key = act ? keys[i] : 0ull; const uint32_t val = act ? vals[i] : 0u;
    const uint32_t dig = act ? ((uint32_t)(key >> shift) & 15u) : 16u;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, dig);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (threadIdx.x < 8 * 17) (&wcnt[0][0])[threadIdx.x] = 0;
    __syncthreads();
    if (rank == 0) wcnt[warp][dig] = __popc(peers);
    __syncthreads();
    if (act) {
        uint32_t off = hist[dig * nblocks + blockIdx.x];
        for (uint32_t w = 0; w < warp; w++) off += wcnt[w][dig];
        keys_out[off + rank] = key; vals_out[off + rank] = val;
    }
}

// ---- 4. reorder into Morton order ---------------------------------------------------------------
__global__ void k_reorder(const BvhTri *__restrict__ tmp, const uint32_t *__restrict__ ref_tri, const float *__restrict__ aabb, const uint32_t *__restrict__ vals, uint32_t n,
                          BvhTri *__restrict__ tris, float *__restrict__ leaf_box, uint32_t *__restrict__ tri_slot) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t g = vals[i];
    const BvhTri t = tmp[ref_tri[g]];
    tris[i] = t;
    tri_slot[__float_as_uint(t.a.w)] = i;       // any one of the triangle's reference slots (all hold the same 48 B); benign race
    for (int k = 0; k < 6; k++) leaf_box[(size_t)i * 6 + k] = aabb[(size_t)g * 6 + k];
}

// ---- 5. Karras 2012 hierarchy -------------------------------------------------------------------
__device__ __forceinline__ int lbvh_delta(const unsigned long long *keys, int n, int i, int j) {
    if (j < 0 || j >= n) return -1;
    const unsigned long long a = keys[i], b = keys[j];
    if (a == b) return 64 + __clz((uint32_t)i ^ (uint32_t)j);
    return __clzll((long long)(a ^ b));
}
__global__ void k_karras(const unsigned long long *__restrict__ keys, int n, int *__restrict__ left, int *__restrict__ right, int *__restrict__ parent_int, int *__restrict__ parent_leaf,
                         int2 *__restrict__ range) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const int d = (lbvh_delta(keys, n, i, i + 1) - lbvh_delta(keys, n, i, i - 1)) >= 0 ? 1 : -1;
    const int dmin = lbvh_delta(keys, n, i, i - d);
    int lmax = 2;
    while (lbvh_delta(keys, n, i, i + lmax * d) > dmin) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2) if (lbvh_delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
    const int j = i + l * d;
    const int dnode = lbvh_delta(keys, n, i, j);
    int s = 0;
    for (int t = (l + 1) / 2;; t = (t + 1) / 2) {
        if (lbvh_delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
        if (t <= 1) break;
    }
    const int gamma = i + s * d + min(d, 0);
    const int lo = min(i, j), hi = max(i, j);
    range[i] = make_int2(lo, hi);                                        // triangles (Morton slots) covered by this node
    if (lo == gamma) { left[i] = ~gamma; parent_leaf[gamma] = i; } else { left[i] = gamma; parent_int[gamma] = i; }
    if (hi == gamma + 1) { right[i] = ~(gamma + 1); parent_leaf[gamma + 1] = i; } else { right[i] = gamma + 1; parent_int[gamma + 1] = i; }
    if (i == 0) parent_int[0] = -1;
}

// ---- 6. bottom-up refit ---------------------------------------------------------------------------
__global__ void k_refit(int n, const int *__restrict__ left, const int *__restrict__ right, const int *__restrict__ parent_int, const int *__restrict__ parent_leaf,
                        const float *__restrict__ leaf_box, float *__restrict__ node_box, unsigned int *__restrict__ flags) {
    const int leaf = blockIdx.x * blockDim.x + threadIdx.x;
    if (leaf >= n) return;
    int cur = parent_leaf[leaf];
    while (cur >= 0) {
        if (atomicAdd(&flags[cur], 1u) == 0u) return;                    // first child to arrive stops; second continues
        __threadfence();
        float bx[6];
        const int l = left[cur], r = right[cur];
        const float *a = l < 0 ? leaf_box + (size_t)(~l) * 6 : node_box + (size_t)l * 6;
        const float *b = r < 0 ? leaf_box + (size_t)(~r) * 6 : node_box + (size_t)r * 6;
        for (int k = 0; k < 3; k++) { bx[k] = fminf(__ldcg(a + k), __ldcg(b + k)); bx[3 + k] = fmaxf(__ldcg(a + 3 + k), __ldcg(b + 3 + k)); }
        for (int k = 0; k < 6; k++) __stcg(node_box + (size_t)cur * 6 + k, bx[k]);
        __threadfence();
        cur = parent_int[cur];
    }
}

// ---- 7. emit 64-B nodes (child boxes in the parent, slightly padded so the slab test is conservative) ----
// A subtree covering <= LBVH_LEAF_MAX consecutive Morton slots is referenced as ONE leaf (first slot + count), which removes
// the two deepest levels of the binary hierarchy: fewer node fetches and stack operations per ray.
// leaf reference: child < 0, r = ~child, first = r >> 2, count = (r & 3) + 1
__device__ __forceinline__ int lbvh_child_ref(int c, const int2 *range) {
    if (c < 0) return ~(((~c) << 2) | 0);                                // single triangle
    const int2 r = range[c];
    if (r.y - r.x + 1 <= LBVH_LEAF_MAX) return ~((r.x << 2) | (r.y - r.x));
    return c;
}
// absolute pad: the FMA slab test of bvh_trace perturbs a plane by <= 6e-8*|ray origin|; 2e-6 * (largest |coordinate| of the scene)
// keeps it conservative for origins within ~16 scene extents (every secondary ray), and also covers the rounding of the
// subtract-multiply form, so the traversal needs no slack factor on its interval comparison
__device__ __forceinline__ float scene_pad(const float *bounds) { return bvh_scene_pad(bounds); }
__device__ __forceinline__ void pad_child(const float *box, float pabs, float *lo, float *hi) { bvh_pad_child(box, pabs, lo, hi); }   // box: lo xyz, hi xyz (unpadded)
__global__ void k_emit(int n_int, const int *__restrict__ left, const int *__restrict__ right, const int2 *__restrict__ range, const float *__restrict__ leaf_box,
                       const float *__restrict__ node_box, const float *__restrict__ bounds, BvhNode *__restrict__ nodes) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_int) return;
    const float pabs = scene_pad(bounds);
    const int l = left[i], r = right[i];
    const float *a = l < 0 ? leaf_box + (size_t)(~l) * 6 : node_box + (size_t)l * 6;
    const float *b = r < 0 ? leaf_box + (size_t)(~r) * 6 : node_box + (size_t)r * 6;
    BvhNode nd;
    pad_child(a, pabs, nd.lo0, nd.hi0); pad_child(b, pabs, nd.lo1, nd.hi1);
    nd.c0 = lbvh_child_ref(l, range); nd.c1 = lbvh_child_ref(r, range); nd._pad[0] = nd._pad[1] = 0;
    nodes[i] = nd;
}

// ---- 8. refit after the instance transforms changed (Engine::update_instance_transforms without rebuild) --------------------------------
// Topology, slot order, tri_slot and the shading records stay; every slot's 48-B record, its reference box, every reachable BVH2 child box
// (re-padded from the NEW scene bounds) and the BVH4 child boxes are recomputed.  Deterministic: min / max unions and one fixed arithmetic.
// slot_jk[i] = (j << 16) | k: slot i is slab j of the k slots holding its triangle (k == 1: the whole triangle box).
__global__ void k_refit_slots(const b200pt_vertex *__restrict__ verts, const uint32_t *__restrict__ indices, const DevMesh *__restrict__ meshes,
                              const DevInstance *__restrict__ inst, uint32_t n_inst, const uint32_t *__restrict__ slot_jk, uint32_t n,
                              BvhTri *__restrict__ tris, float *__restrict__ slot_box, float *__restrict__ bounds) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    float lo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, hi[3] = { -3.0e38f, -3.0e38f, -3.0e38f };
    if (i < n) {
        const uint32_t gid = __float_as_uint(tris[i].a.w);
        const uint32_t a = instance_of(inst, n_inst, gid);
        const DevInstance &in = inst[a];
        const uint32_t prim = gid - in.tri_base;
        const DevMesh m = meshes[in.mesh];
        const uint32_t *ix = indices + m.ibase + (size_t)prim * 3;
        float bb[6];
        const BvhTri t = world_tri(in, a, gid, prim, verts[m.vbase + ix[0]], verts[m.vbase + ix[1]], verts[m.vbase + ix[2]], bb);
        tris[i] = t;
        const uint32_t jk = slot_jk[i], k = jk & 0xFFFFu;
        float *o = slot_box + (size_t)i * 6;
        if (k <= 1) { for (int q = 0; q < 6; q++) o[q] = bb[q]; }
        else slab_ref_box(t, bb, jk >> 16, k, o);
        for (int q = 0; q < 3; q++) { lo[q] = bb[q]; hi[q] = bb[3 + q]; }
    }
    reduce_bounds(lo, hi, bounds);
}
// One level of the BVH2 (nodes order[first, first + count), all at the same depth), deepest level first: child boxes from the slot boxes of
// a leaf reference or from node_box of an inner child (written by the level below), padded as k_emit pads them; node_box[node] = the union.
__global__ void k_refit_level(const int32_t *__restrict__ order, uint32_t first, uint32_t count, const float *__restrict__ slot_box,
                              const float *__restrict__ bounds, BvhNode *__restrict__ nodes, float *__restrict__ node_box) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int32_t n = order[first + i];
    BvhNode nd = nodes[n];
    const float pabs = scene_pad(bounds);
    float u[6] = { 3.0e38f, 3.0e38f, 3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f };
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const int32_t c = s ? nd.c1 : nd.c0;
        float box[6] = { 3.0e38f, 3.0e38f, 3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f };
        if (c < 0) {                                                      // leaf: slots [first, first + count)
            const uint32_t r = (uint32_t)(~c), f = r >> 2, cnt = (r & 3u) + 1u;
            for (uint32_t q = f; q < f + cnt; q++)
                for (int k = 0; k < 3; k++) { box[k] = fminf(box[k], slot_box[(size_t)q * 6 + k]); box[3 + k] = fmaxf(box[3 + k], slot_box[(size_t)q * 6 + 3 + k]); }
        } else {
            for (int k = 0; k < 6; k++) box[k] = __ldcg(node_box + (size_t)c * 6 + k);
        }
        pad_child(box, pabs, s ? nd.lo1 : nd.lo0, s ? nd.hi1 : nd.hi0);
        for (int k = 0; k < 3; k++) { u[k] = fminf(u[k], box[k]); u[3 + k] = fmaxf(u[3 + k], box[3 + k]); }
    }
    nodes[n] = nd;
    for (int k = 0; k < 6; k++) __stcg(node_box + (size_t)n * 6 + k, u[k]);
}
// BVH4 child boxes: bvh4_collapse_host copies every BVH4 child box verbatim from one BVH2 child box; src[4 * node4 + k] names it
// ((BVH2 node << 1) | side, or -1 for an empty slot), so the refit BVH4 is exactly as conservative as the refit BVH2.
__global__ void k_refit_wide(const int32_t *__restrict__ src, uint32_t n4, const BvhNode *__restrict__ nodes2, Bvh4Node *__restrict__ nodes4) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4 * 4u) return;
    const int32_t s = src[i];
    if (s < 0) return;
    const BvhNode &N = nodes2[s >> 1];
    const float *lo = (s & 1) ? N.lo1 : N.lo0, *hi = (s & 1) ? N.hi1 : N.hi0;
    Bvh4Node &o = nodes4[i >> 2]; const uint32_t k = i & 3u;
    o.lox[k] = lo[0]; o.loy[k] = lo[1]; o.loz[k] = lo[2]; o.hix[k] = hi[0]; o.hiy[k] = hi[1]; o.hiz[k] = hi[2];
}

// ---- 9. after the mesh vertices changed (Engine::update_mesh_vertices without rebuild) ------------------------------------------------------
// The refit above recomputes the slot records; the shading records (gid order) of the instances of the changed meshes are rewritten here with
// shade_tri, as k_world_tris writes them.  list = [instance ids (m) | prefix of their triangle counts (m + 1)]: one thread per triangle.
__global__ void k_refresh_shade(const b200pt_vertex *__restrict__ verts, const uint32_t *__restrict__ indices, const DevMesh *__restrict__ meshes,
                                const DevInstance *__restrict__ inst, const uint32_t *__restrict__ list, uint32_t m, ShadeTri *__restrict__ shade) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t *off = list + m;
    if (t >= off[m]) return;
    uint32_t lo = 0, hi = m - 1;                                         // last range with off <= t
    while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (off[mid] <= t) lo = mid; else hi = mid - 1; }
    const uint32_t a = list[lo], prim = t - off[lo];
    const DevInstance &in = inst[a];
    const DevMesh msh = meshes[in.mesh];
    const uint32_t *ix = indices + msh.ibase + (size_t)prim * 3;
    shade[in.tri_base + prim] = shade_tri(a, prim, in.material, verts[msh.vbase + ix[0]], verts[msh.vbase + ix[1]], verts[msh.vbase + ix[2]]);
}
// *flag = 1 when any of v[0, n) is not finite (the caller zeroes it first).
__global__ void k_flag_nonfinite(const float *__restrict__ v, size_t n, uint32_t *__restrict__ flag) {
    bool bad = false;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) bad |= !isfinite(v[i]);
    if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) *flag = 1u;
}

// ------------------------------------------------------------------------------------------------
// BVH2 -> BVH4 collapse (host).  Every BVH4 node takes a BVH2 node, starts from its two children and keeps replacing the internal
// child of largest surface area by that child's two children until four slots are filled (or only leaves remain).  Child boxes are
// copied verbatim from the BVH2 nodes, so the BVH4 is exactly as conservative as the BVH2 (same padded boxes, same leaves): both
// structures return identical hits.  Nodes are emitted in breadth-first order (the hot top levels are contiguous).
// ------------------------------------------------------------------------------------------------
// src (optional, 4 entries per BVH4 node): the BVH2 child box each BVH4 child box was copied from, (BVH2 node << 1) | side, -1 when empty
static uint32_t bvh4_collapse_src(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, Bvh4Node *out, int *depth4, int32_t *src) {
    if (depth4) *depth4 = 0;
    if (root2 < 0 || n_nodes2 == 0) return 0;
    struct Slot { int32_t child, src; float lo[3], hi[3]; };
    auto area = [](const Slot &s) { return bvh4_slot_area(s.lo, s.hi); };   // ploc.cu's device collapse ranks by the same bits
    bool bad = false;                                                       // a child index outside the array or a cycle: not a tree
    auto slots_of = [&](int32_t n, Slot &a, Slot &b) {
        if ((uint32_t)n >= n_nodes2) { bad = true; n = 0; }
        const BvhNode &N = nodes2[n];
        a.child = N.c0; b.child = N.c1; a.src = n * 2; b.src = n * 2 + 1;
        for (int k = 0; k < 3; k++) { a.lo[k] = N.lo0[k]; a.hi[k] = N.hi0[k]; b.lo[k] = N.lo1[k]; b.hi[k] = N.hi1[k]; }
    };
    std::vector<std::pair<int32_t, int>> queue;                          // (BVH2 node, depth) of BVH4 node i, in emission order
    queue.reserve(n_nodes2 / 2 + 1);
    queue.push_back({ root2, 1 });
    int max_d = 1;
    for (size_t i = 0; i < queue.size(); i++) {
        if (bad || queue.size() > (size_t)n_nodes2) { if (depth4) *depth4 = 0; return 0; }   // every BVH4 node consumes at least one BVH2 node
        const int32_t n2 = queue[i].first; const int dep = queue[i].second;
        if (dep > max_d) max_d = dep;
        Slot sl[4]; int ns = 2;
        slots_of(n2, sl[0], sl[1]);
        while (ns < 4) {
            int best = -1; float best_a = -1.0f;
            for (int k = 0; k < ns; k++) if (sl[k].child >= 0) { const float a = area(sl[k]); if (a > best_a) { best_a = a; best = k; } }
            if (best < 0) break;
            Slot a, b; slots_of(sl[best].child, a, b);
            sl[best] = a; sl[ns++] = b;
        }
        Bvh4Node &o = out[i];
        for (int k = 0; k < 4; k++) {
            if (k < ns) {
                o.lox[k] = sl[k].lo[0]; o.loy[k] = sl[k].lo[1]; o.loz[k] = sl[k].lo[2];
                o.hix[k] = sl[k].hi[0]; o.hiy[k] = sl[k].hi[1]; o.hiz[k] = sl[k].hi[2];
                if (sl[k].child >= 0) { o.child[k] = (int32_t)queue.size(); queue.push_back({ sl[k].child, dep + 1 }); }
                else o.child[k] = sl[k].child;
            } else {
                o.lox[k] = o.loy[k] = o.loz[k] = o.hix[k] = o.hiy[k] = o.hiz[k] = 3.0e38f;
                o.child[k] = BVH4_EMPTY;
            }
            o._pad[k] = 0;
            if (src) src[i * 4 + k] = k < ns ? sl[k].src : -1;
        }
    }
    if (bad || queue.size() > (size_t)n_nodes2) { if (depth4) *depth4 = 0; return 0; }
    if (depth4) *depth4 = max_d;
    return (uint32_t)queue.size();
}
uint32_t bvh4_collapse_host(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, Bvh4Node *out, int *depth4) {
    return bvh4_collapse_src(nodes2, n_nodes2, root2, out, depth4, nullptr);
}

// ------------------------------------------------------------------------------------------------
// Tree-quality passes on the host (OPT-IN: B200PT_BVH_SAH=1 or 2, see Engine::upload_scene and lbvh_refine_sah).
// DESIGN.md section 9 item 1a: the traversal kernels are bound by the number of node / triangle visits of the Morton-order tree, not by their
// loop shape.  Both passes build top-down with a 16-bin surface-area heuristic over box centroids (cost = area x references on each side,
// all three axes tried, median split in index order when the bins cannot separate the items) and emit nodes depth-first with root 0.
//   bvh2_sah_rebuild_host  (mode 1): the LBVH's leaves (<= 4 consecutive slots, with the padded boxes stored for them) are kept; only the
//                          inner nodes above them are rebuilt.  Child boxes are exact unions of leaf boxes: same hits, triangle order untouched.
//   bvh2_sah_build_host    (mode 2): built from the per-slot reference boxes; leaves are re-formed (<= 4 references, a small range stays a
//                          leaf when that is cheaper than splitting it), which permutes the reference slots (perm[new slot] = old slot).
// ------------------------------------------------------------------------------------------------
namespace {
struct SahItem { int32_t ref; uint32_t count; float lo[3], hi[3], c[3]; };
inline double sah_area(const float lo[3], const float hi[3]) { const double dx = (double)hi[0] - lo[0], dy = (double)hi[1] - lo[1], dz = (double)hi[2] - lo[2]; return 2.0 * (dx * dy + dy * dz + dz * dx); }
inline void sah_bounds(const std::vector<SahItem> &it, uint32_t b, uint32_t e, float lo[3], float hi[3]) {
    for (int a = 0; a < 3; a++) { lo[a] = 3.0e38f; hi[a] = -3.0e38f; }
    for (uint32_t i = b; i < e; i++) for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], it[i].lo[a]); hi[a] = fmaxf(hi[a], it[i].hi[a]); }
}
// Partitions it[b, e) in place and returns mid (b < mid < e).  *cost = area(left) x count(left) + area(right) x count(right) of the split taken.
uint32_t sah_split(std::vector<SahItem> &it, uint32_t b, uint32_t e, double *cost) {
    constexpr int NB = 16;
    float clo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, chi[3] = { -3.0e38f, -3.0e38f, -3.0e38f };
    for (uint32_t i = b; i < e; i++) for (int a = 0; a < 3; a++) { clo[a] = fminf(clo[a], it[i].c[a]); chi[a] = fmaxf(chi[a], it[i].c[a]); }
    int best_axis = -1, best_bin = -1; double best_cost = 1e300;
    for (int a = 0; a < 3; a++) {
        const float ext = chi[a] - clo[a];
        if (!(ext > 0.0f)) continue;
        float blo[NB][3], bhi[NB][3]; uint32_t bcnt[NB];
        for (int k = 0; k < NB; k++) { bcnt[k] = 0; for (int q = 0; q < 3; q++) { blo[k][q] = 3.0e38f; bhi[k][q] = -3.0e38f; } }
        const float scale = (float)NB / ext;
        for (uint32_t i = b; i < e; i++) {
            int k = (int)((it[i].c[a] - clo[a]) * scale); if (k >= NB) k = NB - 1; if (k < 0) k = 0;
            bcnt[k] += it[i].count;
            for (int q = 0; q < 3; q++) { blo[k][q] = fminf(blo[k][q], it[i].lo[q]); bhi[k][q] = fmaxf(bhi[k][q], it[i].hi[q]); }
        }
        double rarea[NB]; uint32_t rcnt[NB];
        { float lo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, hi[3] = { -3.0e38f, -3.0e38f, -3.0e38f }; uint32_t c = 0;
          for (int k = NB - 1; k >= 1; k--) { if (bcnt[k]) for (int q = 0; q < 3; q++) { lo[q] = fminf(lo[q], blo[k][q]); hi[q] = fmaxf(hi[q], bhi[k][q]); } c += bcnt[k]; rcnt[k] = c; rarea[k] = c ? sah_area(lo, hi) : 0.0; } }
        float lo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, hi[3] = { -3.0e38f, -3.0e38f, -3.0e38f }; uint32_t c = 0;
        for (int k = 0; k < NB - 1; k++) {                                  // split between bin k and k + 1
            if (bcnt[k]) for (int q = 0; q < 3; q++) { lo[q] = fminf(lo[q], blo[k][q]); hi[q] = fmaxf(hi[q], bhi[k][q]); }
            c += bcnt[k];
            if (!c || !rcnt[k + 1]) continue;
            const double cst = sah_area(lo, hi) * c + rarea[k + 1] * rcnt[k + 1];
            if (cst < best_cost) { best_cost = cst; best_axis = a; best_bin = k; }
        }
    }
    uint32_t mid = b;
    if (best_axis >= 0) {
        const float ext = chi[best_axis] - clo[best_axis], scale = (float)NB / ext;
        auto bin_of = [&](const SahItem &L) { int k = (int)((L.c[best_axis] - clo[best_axis]) * scale); if (k >= NB) k = NB - 1; if (k < 0) k = 0; return k; };
        mid = (uint32_t)(std::partition(it.begin() + b, it.begin() + e, [&](const SahItem &L) { return bin_of(L) <= best_bin; }) - it.begin());
    }
    if (mid == b || mid == e) {                                             // identical centroids: median split in index order
        mid = b + (e - b) / 2;
        float lo[3], hi[3]; uint32_t cl = 0, cr = 0;
        for (uint32_t i = b; i < mid; i++) cl += it[i].count;
        for (uint32_t i = mid; i < e; i++) cr += it[i].count;
        sah_bounds(it, b, mid, lo, hi); best_cost = sah_area(lo, hi) * cl; sah_bounds(it, mid, e, lo, hi); best_cost += sah_area(lo, hi) * cr;
    }
    if (cost) *cost = best_cost;
    return mid;
}
// Top-down build of items [0, n) on a pool of host threads.  A subtree over k items emits at most k - 1 nodes, so node `me` over [b, e) keeps
// its left subtree in the block starting at me + 1 and its right subtree in the block starting at me + (mid - b): every index is known
// before the subtree is built, ranges of >= 1024 items go through a shared queue, smaller ones are finished by the thread that produced
// them (disjoint item ranges, disjoint output blocks).  With `used` == nullptr the blocks are exact (k items -> k - 1 nodes); otherwise
// used[i] marks the nodes written and the caller compacts the array (block order == depth-first order, so compaction keeps the layout).
// The result does not depend on the thread count or the schedule.  P: bool leaf(x, y) / int32_t ref(x, y) / void box(x, y, lo, hi).
template <class P>
void sah_pool_build(std::vector<SahItem> &it, uint32_t n_items, BvhNode *out, uint8_t *used, P &pol) {
    struct Range { uint32_t b, e, me; };
    unsigned n_threads = std::thread::hardware_concurrency(); if (n_threads == 0) n_threads = 1;
    if (const char *e = getenv("B200PT_HOST_THREADS")) { const int v = atoi(e); if (v >= 1) n_threads = (unsigned)v; }
    if (n_threads > 64) n_threads = 64;
    if (n_items < 8192) n_threads = 1;
    std::mutex mtx; std::condition_variable cv; std::vector<Range> shared{ { 0, n_items, 0 } }; int active = 0;
    auto worker = [&]() {
        std::vector<Range> local;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(mtx);
                cv.wait(lk, [&] { return !shared.empty() || active == 0; });
                if (shared.empty()) return;                                    // nothing queued and nobody working: done
                local.push_back(shared.back()); shared.pop_back(); active++;
            }
            while (!local.empty()) {
                const Range t = local.back(); local.pop_back();
                const uint32_t mid = sah_split(it, t.b, t.e, nullptr);
                BvhNode &N = out[t.me]; N._pad[0] = N._pad[1] = 0;
                if (used) used[t.me] = 1;
                pol.box(t.b, mid, N.lo0, N.hi0); pol.box(mid, t.e, N.lo1, N.hi1);
                const uint32_t left_me = t.me + 1, right_me = t.me + (mid - t.b);
                const bool left_leaf = pol.leaf(t.b, mid), right_leaf = pol.leaf(mid, t.e);
                N.c0 = left_leaf ? pol.ref(t.b, mid) : (int32_t)left_me;
                N.c1 = right_leaf ? pol.ref(mid, t.e) : (int32_t)right_me;
                const Range kid[2] = { { mid, t.e, right_me }, { t.b, mid, left_me } };   // left last: depth-first within a thread
                const bool is_leaf[2] = { right_leaf, left_leaf };
                for (int k = 0; k < 2; k++) {
                    if (is_leaf[k]) continue;
                    if (n_threads > 1 && kid[k].e - kid[k].b >= 1024) { { std::lock_guard<std::mutex> lk(mtx); shared.push_back(kid[k]); } cv.notify_one(); }
                    else local.push_back(kid[k]);
                }
            }
            { std::lock_guard<std::mutex> lk(mtx); active--; }
            cv.notify_all();
        }
    };
    std::vector<std::thread> pool;
    for (unsigned i = 1; i < n_threads; i++) { try { pool.emplace_back(worker); } catch (...) { break; } }   // no thread to be had: fewer workers
    worker();
    for (auto &th : pool) th.join();
}
// depth and SAH cost (unnormalised) of a tree whose children follow their parents: one forward sweep
void tree_depth_cost(const BvhNode *out, uint32_t n_out, int *max_d, double *cost) {
    std::vector<int> dep(n_out, 0); dep[0] = 1; *max_d = 1; *cost = 0.0;
    for (uint32_t i = 0; i < n_out; i++) {
        const BvhNode &N = out[i];
        if (dep[i] > *max_d) *max_d = dep[i];
        for (int k = 0; k < 2; k++) {
            const int32_t c = k ? N.c1 : N.c0; const double a = sah_area(k ? N.lo1 : N.lo0, k ? N.hi1 : N.hi0);
            if (c >= 0) { dep[c] = dep[i] + 1; *cost += a; } else *cost += a * (double)(((uint32_t)(~c) & 3u) + 1u);
        }
    }
}
} // namespace

// Returns the node count (leaves - 1; 0 if the root is a leaf or the input is not a tree), *depth = new depth, sah[0/1] = SAH cost before / after.
uint32_t bvh2_sah_rebuild_host(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, BvhNode *out, int *depth, double sah[2]) {
    if (depth) *depth = 0;
    if (sah) sah[0] = sah[1] = 0.0;
    if (root2 < 0 || n_nodes2 == 0 || (uint32_t)root2 >= n_nodes2) return 0;
    std::vector<SahItem> leaves; leaves.reserve(n_nodes2 + 1);
    double cost_in = 0.0;
    {   // collect the leaves (and the SAH cost of the input tree, relative to the root box)
        std::vector<int32_t> stack{ root2 }; size_t visited = 0;
        while (!stack.empty()) {
            const int32_t n = stack.back(); stack.pop_back();
            if ((uint32_t)n >= n_nodes2 || ++visited > (size_t)n_nodes2) return 0;             // not a tree
            const BvhNode &N = nodes2[n];
            for (int k = 0; k < 2; k++) {
                const int32_t c = k ? N.c1 : N.c0; const float *lo = k ? N.lo1 : N.lo0, *hi = k ? N.hi1 : N.hi0;
                if (c >= 0) { cost_in += sah_area(lo, hi); stack.push_back(c); }
                else {
                    SahItem L; L.ref = c; L.count = ((uint32_t)(~c) & 3u) + 1u;
                    for (int a = 0; a < 3; a++) { L.lo[a] = lo[a]; L.hi[a] = hi[a]; L.c[a] = 0.5f * (lo[a] + hi[a]); }
                    cost_in += sah_area(lo, hi) * L.count;
                    leaves.push_back(L);
                }
            }
        }
    }
    const uint32_t nl = (uint32_t)leaves.size();
    if (nl < 2 || nl - 1 > n_nodes2) return 0;
    struct KeepLeaves {                                                     // the LBVH's leaves stay as they are: k leaves -> exactly k - 1 nodes
        std::vector<SahItem> &it;
        bool leaf(uint32_t x, uint32_t y) { return y - x == 1; }
        int32_t ref(uint32_t x, uint32_t) { return it[x].ref; }
        void box(uint32_t x, uint32_t y, float *lo, float *hi) { sah_bounds(it, x, y, lo, hi); }
    } pol{ leaves };
    sah_pool_build(leaves, nl, out, nullptr, pol);
    const uint32_t n_out = nl - 1; int max_d = 1; double cost_out = 0.0;
    tree_depth_cost(out, n_out, &max_d, &cost_out);
    if (depth) *depth = max_d;
    if (sah) { float lo[3], hi[3]; sah_bounds(leaves, 0, nl, lo, hi); const double ra = sah_area(lo, hi); sah[0] = ra > 0 ? cost_in / ra : 0.0; sah[1] = ra > 0 ? cost_out / ra : 0.0; }
    return n_out;
}

// Insertion-based refinement (after Bittner, Hapala, Havran 2013, "Fast insertion-based optimization of bounding volume hierarchies"):
// the nodes of largest surface area are taken out of the tree one at a time (the sibling takes the parent's place) and put back at the
// position that adds the least surface area, found by a branch-and-bound descent from the root.  Leaves (references and their stored,
// padded boxes) are untouched, inner boxes are unions of leaf boxes: same hits.  `passes` sweeps over the `fraction` largest nodes each.
// Output as in bvh2_sah_rebuild_host (depth-first, root 0, same node count).  Returns 0 when the input is not a tree or has < 3 leaves.
uint32_t bvh2_reinsert_host(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, BvhNode *out, int passes, float fraction, int *depth, double sah[2]) {
    if (depth) *depth = 0;
    if (sah) sah[0] = sah[1] = 0.0;
    if (root2 < 0 || n_nodes2 == 0 || (uint32_t)root2 >= n_nodes2 || !out) return 0;
    struct T { float lo[3], hi[3]; int parent, c[2]; int32_t ref; float area; };   // leaves: c = {-1, -1}, ref < 0
    std::vector<T> t; t.reserve(2 * (size_t)n_nodes2 + 1);
    auto set_area = [](T &x) { x.area = (float)sah_area(x.lo, x.hi); };
    {   // pointer tree with a box per node; element 0 is the root
        struct E { int32_t n2; int parent; int side; };
        std::vector<E> stack{ { root2, -1, 0 } }; size_t visited = 0;
        while (!stack.empty()) {
            const E e = stack.back(); stack.pop_back();
            if ((uint32_t)e.n2 >= n_nodes2 || ++visited > (size_t)n_nodes2) return 0;
            const BvhNode &N = nodes2[e.n2];
            const int me = (int)t.size(); t.push_back(T{});
            t[me].parent = e.parent; t[me].ref = 0; t[me].c[0] = t[me].c[1] = -1;
            for (int a = 0; a < 3; a++) { t[me].lo[a] = fminf(N.lo0[a], N.lo1[a]); t[me].hi[a] = fmaxf(N.hi0[a], N.hi1[a]); }
            set_area(t[me]);
            if (e.parent >= 0) t[e.parent].c[e.side] = me;
            for (int k = 0; k < 2; k++) {
                const int32_t c = k ? N.c1 : N.c0;
                if (c >= 0) stack.push_back({ c, me, k });
                else {
                    const int lf = (int)t.size(); t.push_back(T{});
                    t[lf].parent = me; t[lf].ref = c; t[lf].c[0] = t[lf].c[1] = -1; t[me].c[k] = lf;
                    for (int a = 0; a < 3; a++) { t[lf].lo[a] = k ? N.lo1[a] : N.lo0[a]; t[lf].hi[a] = k ? N.hi1[a] : N.hi0[a]; }
                    set_area(t[lf]);
                }
            }
        }
    }
    const uint32_t n_all = (uint32_t)t.size(), n_inner = n_all / 2;            // a full binary tree: inner = leaves - 1
    if (n_all < 5 || n_inner > n_nodes2) return 0;
    auto weight = [&](const T &x) { return x.c[0] < 0 ? (double)(((uint32_t)(~x.ref) & 3u) + 1u) : 1.0; };
    auto cost = [&]() { double c = 0.0; for (uint32_t i = 1; i < n_all; i++) c += (double)t[i].area * weight(t[i]); return c; };
    int root = 0;
    const double root_area = t[0].area, cost_in = cost();
    auto refit_up = [&](int n) {
        while (n >= 0) {
            T &x = t[n]; const T &a = t[x.c[0]], &b = t[x.c[1]];
            bool same = true;
            for (int k = 0; k < 3; k++) {
                const float lo = fminf(a.lo[k], b.lo[k]), hi = fmaxf(a.hi[k], b.hi[k]);
                if (lo != x.lo[k] || hi != x.hi[k]) same = false;
                x.lo[k] = lo; x.hi[k] = hi;
            }
            if (same) break;
            set_area(x); n = x.parent;
        }
    };
    auto union_area = [&](const T &a, const T &b) {
        float lo[3], hi[3];
        for (int k = 0; k < 3; k++) { lo[k] = fminf(a.lo[k], b.lo[k]); hi[k] = fmaxf(a.hi[k], b.hi[k]); }
        return (float)sah_area(lo, hi);
    };
    std::vector<std::pair<float, int>> heap;                                  // (-induced cost, node): std::push_heap keeps the smallest induced cost on top
    std::vector<std::pair<float, int>> cand;
    for (int pass = 0; pass < passes; pass++) {
        cand.clear();
        for (uint32_t i = 0; i < n_all; i++) if ((int)i != root && t[i].parent != root) cand.push_back({ t[i].area, (int)i });
        const size_t take = std::min(cand.size(), (size_t)((double)cand.size() * fraction) + 1);
        std::partial_sort(cand.begin(), cand.begin() + take, cand.end(), [](const std::pair<float, int> &a, const std::pair<float, int> &b) { return a.first > b.first || (a.first == b.first && a.second < b.second); });
        for (size_t ci = 0; ci < take; ci++) {
            const int n = cand[ci].second, p = t[n].parent;
            if (n == root || p < 0 || p == root) continue;                      // the tree changes under the sweep
            const int g = t[p].parent, sib = t[p].c[0] == n ? t[p].c[1] : t[p].c[0];
            // take n (and its parent p) out: the sibling moves up
            t[g].c[t[g].c[0] == p ? 0 : 1] = sib; t[sib].parent = g;
            refit_up(g);
            // branch and bound for the cheapest position
            int best = sib; float best_cost = 3.0e38f;
            heap.clear(); heap.push_back({ -0.0f, root });
            const float na = t[n].area;
            int budget = 8192;                                                  // bounds the search on pathological (heavily overlapping) scenes; any stop leaves a valid tree
            while (!heap.empty() && budget-- > 0) {
                std::pop_heap(heap.begin(), heap.end()); const float induced = -heap.back().first; const int x = heap.back().second; heap.pop_back();
                if (induced + na >= best_cost) break;
                const float direct = union_area(t[x], t[n]), total = induced + direct;
                if (total < best_cost) { best_cost = total; best = x; }
                const float child_induced = total - t[x].area;
                if (t[x].c[0] >= 0 && child_induced + na < best_cost) {
                    heap.push_back({ -child_induced, t[x].c[0] }); std::push_heap(heap.begin(), heap.end());
                    heap.push_back({ -child_induced, t[x].c[1] }); std::push_heap(heap.begin(), heap.end());
                }
            }
            // put it back: p becomes the parent of (best, n)
            const int bp = t[best].parent;
            t[p].parent = bp; t[p].c[0] = best; t[p].c[1] = n; t[best].parent = p; t[n].parent = p;
            if (bp >= 0) t[bp].c[t[bp].c[0] == best ? 0 : 1] = p; else root = p;
            for (int k = 0; k < 3; k++) { t[p].lo[k] = 3.0e38f; t[p].hi[k] = -3.0e38f; }      // force the refit to start here
            refit_up(p);
        }
    }
    // emit depth-first from the (possibly new) root
    struct Task { int n; int32_t parent; int side; int dep; };
    std::vector<Task> tasks{ { root, -1, 0, 1 } };
    uint32_t n_out = 0; int max_d = 1; double cost_out = 0.0;
    while (!tasks.empty()) {
        const Task k = tasks.back(); tasks.pop_back();
        const uint32_t me = n_out++;
        if (me >= n_nodes2) return 0;
        BvhNode &N = out[me]; N._pad[0] = N._pad[1] = 0;
        if (k.parent >= 0) { if (k.side) out[k.parent].c1 = (int32_t)me; else out[k.parent].c0 = (int32_t)me; }
        if (k.dep > max_d) max_d = k.dep;
        const T &a = t[t[k.n].c[0]], &b = t[t[k.n].c[1]];
        for (int q = 0; q < 3; q++) { N.lo0[q] = a.lo[q]; N.hi0[q] = a.hi[q]; N.lo1[q] = b.lo[q]; N.hi1[q] = b.hi[q]; }
        cost_out += (double)a.area * weight(a) + (double)b.area * weight(b);
        if (b.c[0] >= 0) tasks.push_back({ t[k.n].c[1], (int32_t)me, 1, k.dep + 1 }); else N.c1 = b.ref;
        if (a.c[0] >= 0) tasks.push_back({ t[k.n].c[0], (int32_t)me, 0, k.dep + 1 }); else N.c0 = a.ref;
    }
    if (depth) *depth = max_d;
    if (sah) { sah[0] = root_area > 0 ? cost_in / root_area : 0.0; sah[1] = root_area > 0 ? cost_out / root_area : 0.0; }
    return n_out;
}

// ref_boxes: n x 6 floats (lo xyz, hi xyz) per reference slot, unpadded.  out: room for n - 1 nodes; perm: n entries, perm[new slot] = old slot.
// Child boxes get k_emit's padding (4e-7 relative + 2e-6 x the largest |coordinate| of the scene), so the FMA slab test stays conservative.
// trav_cost: price of one node visit in units of one triangle test (1.0: the classic SAH; larger keeps bigger leaves).
// Returns the node count (0 when n <= LBVH_LEAF_MAX: the whole scene is one leaf and the caller keeps what it has); *sah_cost relative to the root box.
uint32_t bvh2_sah_build_host(const float *ref_boxes, uint32_t n, float trav_cost, BvhNode *out, uint32_t *perm, int *depth, double *sah_cost) {
    if (depth) *depth = 0;
    if (sah_cost) *sah_cost = 0.0;
    if (!ref_boxes || !out || !perm || n <= (uint32_t)LBVH_LEAF_MAX || n >= (1u << 28)) return 0;   // leaf references keep the slot in 28 bits
    std::vector<SahItem> it(n);
    float ext = 0.0f;
    for (uint32_t i = 0; i < n; i++) {
        SahItem &I = it[i]; I.ref = (int32_t)i; I.count = 1;
        for (int a = 0; a < 3; a++) {
            I.lo[a] = ref_boxes[(size_t)i * 6 + a]; I.hi[a] = ref_boxes[(size_t)i * 6 + 3 + a]; I.c[a] = 0.5f * (I.lo[a] + I.hi[a]);
            if (!(I.lo[a] <= I.hi[a])) return 0;                            // NaN or inverted box
            ext = fmaxf(ext, fmaxf(fabsf(I.lo[a]), fabsf(I.hi[a])));
        }
    }
    const float pabs = 2e-6f * ext + 1e-30f;
    struct FormLeaves {                                                     // a range of <= LBVH_LEAF_MAX references stays a leaf unless splitting it is cheaper
        std::vector<SahItem> &it; float pabs, trav_cost;
        bool leaf(uint32_t x, uint32_t y) {
            const uint32_t cnt = y - x;
            if (cnt == 1) return true;
            if (cnt > (uint32_t)LBVH_LEAF_MAX) return false;
            float rlo[3], rhi[3]; sah_bounds(it, x, y, rlo, rhi);
            double split_cost; sah_split(it, x, y, &split_cost);               // (reorders inside the range only)
            const double a = sah_area(rlo, rhi);
            return (double)cnt * a <= (double)trav_cost * a + split_cost;
        }
        int32_t ref(uint32_t x, uint32_t y) { return ~(int32_t)((x << 2) | (y - x - 1)); }
        void box(uint32_t x, uint32_t y, float *lo, float *hi) {
            sah_bounds(it, x, y, lo, hi);
            for (int a = 0; a < 3; a++) { const float p = 4e-7f * fmaxf(fabsf(lo[a]), fabsf(hi[a])) + pabs; lo[a] -= p; hi[a] += p; }
        }
    } pol{ it, pabs, trav_cost };
    std::vector<uint8_t> used(n - 1, 0);
    sah_pool_build(it, n, out, used.data(), pol);
    uint32_t n_out = 0;
    {   // compact the blocks (ascending index == depth-first order) and renumber the children
        std::vector<uint32_t> remap(n - 1, 0);
        for (uint32_t i = 0; i + 1 < n; i++) if (used[i]) remap[i] = n_out++;
        for (uint32_t i = 0; i + 1 < n; i++) {
            if (!used[i]) continue;
            BvhNode N = out[i];
            if (N.c0 >= 0) N.c0 = (int32_t)remap[N.c0];
            if (N.c1 >= 0) N.c1 = (int32_t)remap[N.c1];
            out[remap[i]] = N;                                                   // remap[i] <= i: never overwrites a node still to be moved
        }
    }
    int max_d = 1; double cost_out = 0.0;
    tree_depth_cost(out, n_out, &max_d, &cost_out);
    for (uint32_t i = 0; i < n; i++) perm[i] = (uint32_t)it[i].ref;
    if (depth) *depth = max_d;
    if (sah_cost) { float lo[3], hi[3]; sah_bounds(it, 0, n, lo, hi); const double ra = sah_area(lo, hi); *sah_cost = ra > 0 ? cost_out / ra : 0.0; }
    return n_out;
}

// PLOC build from reference boxes in Morton order: the host restatement of ploc.cu's device builder, step for step through the same helpers
// (bvh_build_rules.cuh), so the two give the same nodes, perm and depth bit for bit.  Every reference starts as a cluster; each step, every
// cluster finds its nearest neighbour (ploc_nearest), each mutual pair i < j merges into a new node (left i, right j) that takes position i,
// and the surviving clusters are compacted in order.  Leaves by ploc_leaf_ok (the topmost qualifying node wins), nodes depth-first, left
// first, root 0, child boxes padded by bvh_pad_child with the pad of the references' union.  Conventions and rejections of bvh2_sah_build_host.
uint32_t bvh2_ploc_build_host(const float *ref_boxes, uint32_t n, BvhNode *out, uint32_t *perm, int *depth, double *sah_cost) {
    if (depth) *depth = 0;
    if (sah_cost) *sah_cost = 0.0;
    if (!ref_boxes || !out || !perm || n <= (uint32_t)LBVH_LEAF_MAX || n >= (1u << 28)) return 0;
    for (size_t i = 0; i < (size_t)n; i++)
        for (int a = 0; a < 3; a++) if (!(ref_boxes[i * 6 + a] <= ref_boxes[i * 6 + 3 + a])) return 0;   // NaN or inverted box
    std::vector<float> box((size_t)(2 * n - 1) * 6);
    std::copy(ref_boxes, ref_boxes + (size_t)n * 6, box.begin());
    std::vector<PlocMeta> meta(2 * n - 1, PlocMeta{ 1u, 0u, 0u, 1u });
    std::vector<uint32_t> child(2 * (size_t)(n - 1)), cl(n), nxt, nn(n);
    for (uint32_t i = 0; i < n; i++) cl[i] = i;
    uint32_t next = n;
    while (cl.size() > 1) {
        const uint32_t m = (uint32_t)cl.size();
        for (uint32_t i = 0; i < m; i++) nn[i] = ploc_nearest(cl.data(), m, i, box.data());
        nxt.clear();
        for (uint32_t i = 0; i < m; i++) {
            const uint32_t j = nn[i];
            const bool mutual = nn[j] == i;
            if (mutual && j < i) continue;                                     // merged into position j
            uint32_t id = cl[i];
            if (mutual) { id = next++; ploc_merge(id, cl[i], cl[j], n, box.data(), meta.data(), child.data()); }
            nxt.push_back(id);
        }
        cl.swap(nxt);
    }
    const uint32_t root = cl[0], n_out = meta[root].sub;
    const float pabs = bvh_scene_pad(&box[(size_t)root * 6]);
    struct Task { uint32_t x, idx, first; };
    std::vector<Task> stack{ { root, 0u, 0u } };
    while (!stack.empty()) {
        const Task t = stack.back(); stack.pop_back();
        uint32_t kid_idx[2], kid_first[2];
        ploc_emit(t.x, t.idx, t.first, n, box.data(), meta.data(), child.data(), pabs, out, perm, kid_idx, kid_first);
        for (int s = 0; s < 2; s++) if (kid_idx[s] != 0xFFFFFFFFu) stack.push_back({ child[2 * (size_t)(t.x - n) + s], kid_idx[s], kid_first[s] });
    }
    if (depth) *depth = (int)meta[root].dep;
    if (sah_cost) {
        int d; double c; tree_depth_cost(out, n_out, &d, &c);
        const float *rb = &box[(size_t)root * 6]; const double ra = sah_area(rb, rb + 3);
        *sah_cost = ra > 0 ? c / ra : 0.0;
    }
    return n_out;
}

int lbvh_build_wide(LbvhResult *r, cudaStream_t st) {
    r->nodes4 = nullptr; r->n_nodes4 = 0; r->depth4 = 0;
    if (!r->nodes || r->root < 0 || r->n_nodes == 0) return 0;
    std::vector<BvhNode> h2(r->n_nodes);
    LBVH_CHECK(cudaMemcpyAsync(h2.data(), r->nodes.get(), (size_t)r->n_nodes * sizeof(BvhNode), cudaMemcpyDeviceToHost, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    std::vector<Bvh4Node> h4(r->n_nodes);
    int d4 = 0;
    const uint32_t n4 = bvh4_collapse_host(h2.data(), r->n_nodes, r->root, h4.data(), &d4);
    if (n4 == 0) return 0;
    LBVH_CHECK(alloc(r->nodes4, (size_t)n4 * sizeof(Bvh4Node)));
    LBVH_CHECK(cudaMemcpyAsync(r->nodes4.get(), h4.data(), (size_t)n4 * sizeof(Bvh4Node), cudaMemcpyHostToDevice, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    r->n_nodes4 = n4; r->depth4 = d4;
    return 0;
}

// Opt-in (B200PT_BVH_SAH=1..5; 3 = 2 followed by bvh2_reinsert_host, 3 passes over the largest quarter of the nodes; 4 = 1 followed by the
// same; 5 = re-insertion alone on the Morton-order tree -- 1, 4 and 5 leave the triangle slots where they are).  Mode 1 rebuilds the inner nodes in place with bvh2_sah_rebuild_host: the live node count is unchanged
// (leaves - 1), so the rebuilt array fits the existing allocation.  Mode 2 builds from the per-slot reference boxes ref_box with
// bvh2_sah_build_host (at most slots - 1 nodes: fits as well), then permutes the 48-B triangle slots to the new leaf order and re-derives
// tri_slot (global triangle id -> one of its slots) from the ids stored in the slots.  Root becomes 0, max_depth the new depth.
// A no-op for one-leaf scenes.
int lbvh_refine_sah(LbvhResult *r, const float *ref_box, cudaStream_t st, double sah[2], int mode) {
    if (sah) sah[0] = sah[1] = 0.0;
    if (!r->nodes || r->root < 0 || r->n_nodes == 0) return 0;
    std::vector<BvhNode> h2(r->n_nodes), out(r->n_nodes);
    LBVH_CHECK(cudaMemcpyAsync(h2.data(), r->nodes.get(), (size_t)r->n_nodes * sizeof(BvhNode), cudaMemcpyDeviceToHost, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    int depth = 0;
    // two sweeps over the largest tenth of the nodes: SAH cost 37.1 -> 34.10 in 0.17 s on BreakfastRoom (8 host threads) against 33.95 in 0.65 s for three sweeps over a quarter
    int ri_passes = 2; float ri_fraction = 0.10f;                              // B200PT_BVH_RI="passes,fraction" overrides (A/B runs)
    if (const char *e = getenv("B200PT_BVH_RI")) { int p = 0; float f = 0.0f; if (sscanf(e, "%d,%f", &p, &f) == 2 && p >= 1 && p <= 16 && f > 0.0f && f <= 1.0f) { ri_passes = p; ri_fraction = f; } }
    auto reinsert = [&](uint32_t n_in, double *cost_after) {                  // modes 3, 4: insertion-based refinement of `out`, result back in `out`
        std::vector<BvhNode> tmp(r->n_nodes); int d2 = 0; double c2[2];
        const uint32_t m = bvh2_reinsert_host(out.data(), n_in, 0, tmp.data(), ri_passes, ri_fraction, &d2, c2);
        if (m == n_in) { std::copy(tmp.begin(), tmp.begin() + m, out.begin()); depth = d2; if (cost_after) *cost_after = c2[1]; }
    };
    // SAH and re-insertion trees of detail nested around a point can be far deeper than the LBVH (tests/test_traversal_queries.py): keep the
    // shallower input rather than make every traversal kernel carry a deeper stack
    auto depth_ok = [&](int d) { return d + 2 <= BVH_STACK_MAX || d <= r->max_depth; };
    const bool full = mode == 2 || mode == 3, refine = mode >= 3;
    if (full && ref_box && r->n_tris > (uint32_t)LBVH_LEAF_MAX && r->n_tris - 1 <= r->n_nodes) {
        std::vector<uint32_t> perm(r->n_tris);
        double c_new = 0.0, c_old[2] = { 0.0, 0.0 };
        { std::vector<BvhNode> scratch(r->n_nodes); int d; bvh2_sah_rebuild_host(h2.data(), r->n_nodes, r->root, scratch.data(), &d, c_old); }   // cost of the LBVH, for the log
        const uint32_t n = bvh2_sah_build_host(ref_box, r->n_tris, 1.0f, out.data(), perm.data(), &depth, &c_new);
        if (n != 0 && refine) reinsert(n, &c_new);
        if (n != 0 && c_new < c_old[0] && depth_ok(depth)) {                    // never trade the tree for a costlier one
            std::vector<BvhTri> t_old(r->n_tris), t_new(r->n_tris);
            LBVH_CHECK(cudaMemcpyAsync(t_old.data(), r->tris, (size_t)r->n_tris * sizeof(BvhTri), cudaMemcpyDeviceToHost, st));
            LBVH_CHECK(cudaStreamSynchronize(st));
            std::vector<uint32_t> slot(r->n_prims, 0u);
            for (uint32_t i = 0; i < r->n_tris; i++) {
                t_new[i] = t_old[perm[i]];
                uint32_t gid; memcpy(&gid, &t_new[i].a.w, 4);
                if (gid < r->n_prims) slot[gid] = i;
            }
            LBVH_CHECK(cudaMemcpyAsync(r->tris, t_new.data(), (size_t)r->n_tris * sizeof(BvhTri), cudaMemcpyHostToDevice, st));
            LBVH_CHECK(cudaMemcpyAsync(r->tri_slot.get(), slot.data(), (size_t)r->n_prims * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
            LBVH_CHECK(cudaMemcpyAsync(r->nodes.get(), out.data(), (size_t)n * sizeof(BvhNode), cudaMemcpyHostToDevice, st));
            LBVH_CHECK(cudaStreamSynchronize(st));
            r->root = 0; r->max_depth = depth;
            if (sah) { sah[0] = c_old[0]; sah[1] = c_new; }
            return 0;
        }
    }
    uint32_t n; double cst[2] = { 0.0, 0.0 };
    if (mode == 5) n = bvh2_reinsert_host(h2.data(), r->n_nodes, r->root, out.data(), ri_passes, ri_fraction, &depth, cst);   // the Morton-order tree refined directly
    else {
        n = bvh2_sah_rebuild_host(h2.data(), r->n_nodes, r->root, out.data(), &depth, cst);
        if (n != 0 && refine) reinsert(n, &cst[1]);
    }
    if (n == 0) return 0;
    if (sah) { sah[0] = cst[0]; sah[1] = cst[1] < cst[0] ? cst[1] : cst[0]; }
    if (!(cst[1] < cst[0]) || !depth_ok(depth)) return 0;                      // never trade the tree for a costlier one
    LBVH_CHECK(cudaMemcpyAsync(r->nodes.get(), out.data(), (size_t)n * sizeof(BvhNode), cudaMemcpyHostToDevice, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    r->root = 0; r->max_depth = depth;
    return 0;
}

// What the refit needs of the tree, derived once at the first update (set_scene pays nothing for it): the slots' (j, k), the reachable BVH2
// nodes by depth, and the BVH4's source map.  k = slots holding the triangle; j, the slab a slot stands for, follows where the tree placed the
// slot: the slots of one triangle are ranked by the centre of their leaf's box along the triangle's longest axis (ties: slot order).  Any
// permutation of 0..k-1 covers the triangle; this one keeps the build's slab in every slot whose leaf holds no other slab of its triangle, so
// a refit before anything moved gives back the build's boxes there.
static int lbvh_refit_prepare(const LbvhResult *r, LbvhRefit *s, cudaStream_t st) {
    const uint32_t n = r->n_tris, np = r->n_prims;
    std::vector<BvhTri> ht(n);
    LBVH_CHECK(cudaMemcpyAsync(ht.data(), r->tris, (size_t)n * sizeof(BvhTri), cudaMemcpyDeviceToHost, st));
    std::vector<BvhNode> h2(r->root >= 0 ? r->n_nodes : 0);
    if (!h2.empty()) LBVH_CHECK(cudaMemcpyAsync(h2.data(), r->nodes.get(), (size_t)r->n_nodes * sizeof(BvhNode), cudaMemcpyDeviceToHost, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    std::vector<uint32_t> gid(n), jk(n);
    for (uint32_t i = 0; i < n; i++) { memcpy(&gid[i], &ht[i].a.w, 4); if (gid[i] >= np) gid[i] = 0u; }
    s->level_off.clear(); s->n4 = 0;
    std::vector<float> cen((size_t)n * 3, 0.0f);                               // centre of the box of the leaf holding each slot
    std::vector<int32_t> order;
    if (!h2.empty()) {
        order.push_back(r->root);                                              // breadth-first: each depth is one contiguous range
        s->level_off.push_back(0);
        for (size_t b = 0; b < order.size();) {
            const size_t e = order.size();
            for (size_t i = b; i < e; i++) {
                const BvhNode &N = h2[order[i]];
                for (int c = 0; c < 2; c++) {
                    const int32_t ch = c ? N.c1 : N.c0;
                    if (ch >= 0) { order.push_back(ch); continue; }
                    const uint32_t rr = (uint32_t)(~ch), f = rr >> 2, m = (rr & 3u) + 1u;
                    const float *lo = c ? N.lo1 : N.lo0, *hi = c ? N.hi1 : N.hi0;
                    for (uint32_t q = f; q < f + m && q < n; q++) for (int k = 0; k < 3; k++) cen[(size_t)q * 3 + k] = 0.5f * (lo[k] + hi[k]);
                }
            }
            if (order.size() > r->n_nodes) return (int)cudaErrorInvalidValue;   // not a tree
            s->level_off.push_back((uint32_t)e); b = e;
        }
    }
    {   // slots grouped by triangle (counting sort, slot order inside a group), then ranked along the triangle's longest axis
        std::vector<uint32_t> off(np + 1, 0u), slots(n);
        for (uint32_t i = 0; i < n; i++) off[gid[i] + 1]++;
        for (uint32_t g = 0; g < np; g++) off[g + 1] += off[g];
        std::vector<uint32_t> fill(off.begin(), off.end() - 1);
        for (uint32_t i = 0; i < n; i++) slots[fill[gid[i]]++] = i;
        for (uint32_t g = 0; g < np; g++) {
            uint32_t *b = slots.data() + off[g], *e = slots.data() + off[g + 1];
            const uint32_t k = (uint32_t)(e - b);
            if (k == 0) continue;
            if (k > 1) {
                const BvhTri &t = ht[*b];
                float lo[3], hi[3];
                const float v[3][3] = { { t.a.x, t.a.y, t.a.z }, { t.a.x + t.b.x, t.a.y + t.b.y, t.a.z + t.b.z }, { t.a.x + t.c.x, t.a.y + t.c.y, t.a.z + t.c.z } };
                for (int q = 0; q < 3; q++) { lo[q] = fminf(v[0][q], fminf(v[1][q], v[2][q])); hi[q] = fmaxf(v[0][q], fmaxf(v[1][q], v[2][q])); }
                const float ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
                const int axis = (ex >= ey && ex >= ez) ? 0 : (ey >= ez ? 1 : 2);
                std::stable_sort(b, e, [&](uint32_t x, uint32_t y) { return cen[(size_t)x * 3 + axis] < cen[(size_t)y * 3 + axis]; });
            }
            for (uint32_t j = 0; j < k; j++) jk[b[j]] = (j << 16) | k;
        }
    }
    LBVH_CHECK(alloc(s->slot_jk, (size_t)n * 4));
    LBVH_CHECK(alloc(s->slot_box, (size_t)n * 6 * sizeof(float)));
    LBVH_CHECK(alloc(s->bounds, 6 * sizeof(float)));
    LBVH_CHECK(cudaMemcpyAsync(s->slot_jk.get(), jk.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    if (!h2.empty()) {
        LBVH_CHECK(alloc(s->order, order.size() * 4));
        LBVH_CHECK(alloc(s->node_box, (size_t)r->n_nodes * 6 * sizeof(float)));
        LBVH_CHECK(cudaMemcpyAsync(s->order.get(), order.data(), order.size() * 4, cudaMemcpyHostToDevice, st));
        if (r->nodes4) {                                                     // the collapse is deterministic: re-run on the unchanged BVH2 it was built from
            std::vector<Bvh4Node> h4(r->n_nodes); std::vector<int32_t> src((size_t)r->n_nodes * 4);
            int d4 = 0;
            const uint32_t n4 = bvh4_collapse_src(h2.data(), r->n_nodes, r->root, h4.data(), &d4, src.data());
            if (n4 != r->n_nodes4) return (int)cudaErrorInvalidValue;
            LBVH_CHECK(alloc(s->src4, (size_t)n4 * 4 * 4));
            LBVH_CHECK(cudaMemcpyAsync(s->src4.get(), src.data(), (size_t)n4 * 4 * 4, cudaMemcpyHostToDevice, st));
            s->n4 = n4;
        }
    }
    LBVH_CHECK(cudaStreamSynchronize(st));
    s->ready = true;
    return 0;
}

int lbvh_refit(LbvhResult *r, const b200pt_vertex *d_verts, const uint32_t *d_indices, const DevMesh *d_meshes, const DevInstance *d_instances,
               uint32_t n_instances, cudaStream_t st) {
    if (!r->tris || r->n_tris == 0 || n_instances == 0) return (int)cudaErrorInvalidValue;
    LbvhRefit *s = &r->refit;
    if (!s->ready) {
        const int e = lbvh_refit_prepare(r, s, st);
        if (e != 0) { r->refit = LbvhRefit{}; return e; }
    }
    const uint32_t n = r->n_tris;
    const float binit[6] = { 3.0e38f, 3.0e38f, 3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f };
    LBVH_CHECK(cudaMemcpyAsync(s->bounds.get(), binit, sizeof(binit), cudaMemcpyHostToDevice, st));
    k_refit_slots<<<(n + 255) / 256, 256, 0, st>>>(d_verts, d_indices, d_meshes, d_instances, n_instances, s->slot_jk.get(), n, r->tris, s->slot_box.get(), s->bounds.get());
    for (size_t l = s->level_off.size(); l-- > 1;) {                         // deepest level first
        const uint32_t first = s->level_off[l - 1], count = s->level_off[l] - first;
        k_refit_level<<<(count + 255) / 256, 256, 0, st>>>(s->order.get(), first, count, s->slot_box.get(), s->bounds.get(), r->nodes.get(), s->node_box.get());
    }
    if (s->n4) k_refit_wide<<<(s->n4 * 4 + 255) / 256, 256, 0, st>>>(s->src4.get(), s->n4, r->nodes.get(), r->nodes4.get());
    LBVH_CHECK(cudaGetLastError());
    LBVH_CHECK(cudaStreamSynchronize(st));
    return 0;
}

int lbvh_refresh_shade(LbvhResult *r, const b200pt_vertex *d_verts, const uint32_t *d_indices, const DevMesh *d_meshes, const DevInstance *d_instances,
                       const DevInstance *h_instances, const DevMesh *h_meshes, const uint32_t *insts, uint32_t m, uint32_t *d_list, cudaStream_t st) {
    if (!r->shade) return (int)cudaErrorInvalidValue;
    if (m == 0) return 0;
    std::vector<uint32_t> list(insts, insts + m);
    uint64_t total = 0;
    list.push_back(0u);
    for (uint32_t i = 0; i < m; i++) { total += h_meshes[h_instances[insts[i]].mesh].tri_count; if (total > 0xFFFFFFFFull) return (int)cudaErrorInvalidValue; list.push_back((uint32_t)total); }
    if (total == 0) return 0;
    LBVH_CHECK(cudaMemcpyAsync(d_list, list.data(), list.size() * 4, cudaMemcpyHostToDevice, st));
    k_refresh_shade<<<(uint32_t)((total + 255) / 256), 256, 0, st>>>(d_verts, d_indices, d_meshes, d_instances, d_list, m, r->shade.get());
    LBVH_CHECK(cudaGetLastError());
    LBVH_CHECK(cudaStreamSynchronize(st));
    return 0;
}

int any_nonfinite(const float *d_v, size_t n, uint32_t *d_flag, uint32_t *h_small, cudaStream_t st, bool *any) {
    LBVH_CHECK(cudaMemsetAsync(d_flag, 0, 4, st));
    if (n) k_flag_nonfinite<<<(uint32_t)std::min<size_t>((n + 255) / 256, 1024), 256, 0, st>>>(d_v, n, d_flag);
    LBVH_CHECK(cudaGetLastError());
    LBVH_CHECK(cudaMemcpyAsync(h_small, d_flag, 4, cudaMemcpyDeviceToHost, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    *any = h_small[0] != 0u;
    return 0;
}

int lbvh_build(const b200pt_vertex *d_verts, const uint32_t *d_indices, const DevMesh *d_meshes, const DevInstance *d_instances,
               uint32_t n_instances, uint32_t n_tris, LbvhResult *out, cudaStream_t st, std::vector<float> *host_ref_box, DevPtr<float> *dev_ref_box) {
    if (host_ref_box) host_ref_box->clear();
    if (dev_ref_box) dev_ref_box->reset();
    *out = LbvhResult{};
    if (n_tris == 0 || n_instances == 0) return (int)cudaErrorInvalidValue;
    const uint32_t nt = n_tris, ntblocks = (nt + 255) / 256;

    // ---- per-triangle stage: world-space triangles, shading records (final, gid order), boxes, scene bounds, split counts
    DevPtr<ShadeTri> shade; DevPtr<uint32_t> tri_slot, ksplit, ref_off; DevPtr<BvhTri> tmp; DevPtr<float> aabb, bounds;
    LBVH_CHECK(alloc(shade, (size_t)nt * sizeof(ShadeTri)));
    LBVH_CHECK(alloc(tri_slot, (size_t)nt * sizeof(uint32_t)));
    LBVH_CHECK(alloc(tmp, (size_t)nt * sizeof(BvhTri)));
    LBVH_CHECK(alloc(aabb, (size_t)nt * 6 * sizeof(float)));
    LBVH_CHECK(alloc(bounds, 6 * sizeof(float)));
    LBVH_CHECK(alloc(ksplit, (size_t)nt * 4)); LBVH_CHECK(alloc(ref_off, (size_t)nt * 4));
    const float binit[6] = { 3.0e38f, 3.0e38f, 3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f };
    LBVH_CHECK(cudaMemcpyAsync(bounds.get(), binit, sizeof(binit), cudaMemcpyHostToDevice, st));
    k_world_tris<<<ntblocks, 256, 0, st>>>(d_verts, d_indices, d_meshes, d_instances, n_instances, nt, tmp.get(), shade.get(), aabb.get(), bounds.get());
    k_split_count<<<ntblocks, 256, 0, st>>>(tmp.get(), aabb.get(), bounds.get(), nt, ksplit.get());
    std::vector<uint32_t> hk(nt), hoff(nt);
    LBVH_CHECK(cudaMemcpyAsync(hk.data(), ksplit.get(), (size_t)nt * 4, cudaMemcpyDeviceToHost, st));
    LBVH_CHECK(cudaStreamSynchronize(st));
    uint64_t total = 0; for (uint32_t i = 0; i < nt; i++) { hoff[i] = (uint32_t)total; total += hk[i]; }
    if (total >= (1ull << 28)) return (int)cudaErrorMemoryAllocation;       // leaf references keep the slot in 28 bits
    LBVH_CHECK(cudaMemcpyAsync(ref_off.get(), hoff.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, st));

    // ---- per-reference stage
    const uint32_t n = (uint32_t)total, n_int = n > 1 ? n - 1 : 0, n_nodes_alloc = n_int ? n_int : 1;
    const size_t node_bytes = (size_t)n_nodes_alloc * sizeof(BvhNode), tri_bytes = (size_t)n * sizeof(BvhTri);
    DevPtr<BvhNode> nodes;                                                  // [nodes | tris]
    LBVH_CHECK(alloc(nodes, node_bytes + tri_bytes));
    LBVH_CHECK(cudaMemsetAsync(nodes.get(), 0, node_bytes, st));
    BvhTri *tris = reinterpret_cast<BvhTri *>(nodes.get() + n_nodes_alloc);
    DevPtr<float> ref_box, leaf_box, node_box; DevPtr<uint32_t> ref_tri, vals, vals2, hist; DevPtr<unsigned long long> keys, keys2;
    DevPtr<int> left, right, parent_int, parent_leaf; DevPtr<unsigned int> flags; DevPtr<int2> range;
    const uint32_t nblocks = (n + 255) / 256;
    LBVH_CHECK(alloc(ref_box, (size_t)n * 6 * sizeof(float))); LBVH_CHECK(alloc(ref_tri, (size_t)n * 4));
    LBVH_CHECK(alloc(leaf_box, (size_t)n * 6 * sizeof(float)));
    LBVH_CHECK(alloc(node_box, (size_t)n_nodes_alloc * 6 * sizeof(float)));
    LBVH_CHECK(alloc(keys, (size_t)n * 8)); LBVH_CHECK(alloc(vals, (size_t)n * 4));
    LBVH_CHECK(alloc(keys2, (size_t)n * 8)); LBVH_CHECK(alloc(vals2, (size_t)n * 4));
    LBVH_CHECK(alloc(hist, (size_t)16 * nblocks * 4));
    LBVH_CHECK(alloc(range, (size_t)n_nodes_alloc * sizeof(int2)));
    LBVH_CHECK(alloc(left, (size_t)n_nodes_alloc * 4)); LBVH_CHECK(alloc(right, (size_t)n_nodes_alloc * 4));
    LBVH_CHECK(alloc(parent_int, (size_t)n_nodes_alloc * 4)); LBVH_CHECK(alloc(parent_leaf, (size_t)n * 4));
    LBVH_CHECK(alloc(flags, (size_t)n_nodes_alloc * 4));
    LBVH_CHECK(cudaMemsetAsync(flags.get(), 0, (size_t)n_nodes_alloc * 4, st));
    LBVH_CHECK(cudaMemsetAsync(parent_leaf.get(), 0xFF, (size_t)n * 4, st));

    k_make_refs<<<ntblocks, 256, 0, st>>>(tmp.get(), aabb.get(), ksplit.get(), ref_off.get(), nt, ref_box.get(), ref_tri.get());
    k_morton<<<nblocks, 256, 0, st>>>(ref_box.get(), bounds.get(), n, keys.get(), vals.get());
    for (int pass = 0; pass < 16; pass++) {                              // 62-bit keys, 4-bit digits
        k_radix_hist<<<nblocks, 256, 0, st>>>(keys.get(), n, pass * 4, hist.get(), nblocks);
        k_radix_scan<<<1, 1024, 0, st>>>(hist.get(), 16 * nblocks);
        k_radix_scatter<<<nblocks, 256, 0, st>>>(keys.get(), vals.get(), n, pass * 4, hist.get(), nblocks, keys2.get(), vals2.get());
        std::swap(keys, keys2); std::swap(vals, vals2);
    }
    k_reorder<<<nblocks, 256, 0, st>>>(tmp.get(), ref_tri.get(), ref_box.get(), vals.get(), n, tris, leaf_box.get(), tri_slot.get());
    if (n_int) {
        k_karras<<<(n_int + 255) / 256, 256, 0, st>>>(keys.get(), (int)n, left.get(), right.get(), parent_int.get(), parent_leaf.get(), range.get());
        k_refit<<<nblocks, 256, 0, st>>>((int)n, left.get(), right.get(), parent_int.get(), parent_leaf.get(), leaf_box.get(), node_box.get(), flags.get());
        k_emit<<<(n_int + 255) / 256, 256, 0, st>>>((int)n_int, left.get(), right.get(), range.get(), leaf_box.get(), node_box.get(), bounds.get(), nodes.get());
    }
    LBVH_CHECK(cudaStreamSynchronize(st));
    LBVH_CHECK(cudaGetLastError());

    // depth of the hierarchy actually traversed (one-off, on the host) -> traversal stack size
    int max_depth = 1; int root_ref = n_int ? 0 : ~0;
    if (n_int) {
        std::vector<int> hl(n_int), hr(n_int); std::vector<int2> hrange(n_int);
        LBVH_CHECK(cudaMemcpy(hl.data(), left.get(), (size_t)n_int * 4, cudaMemcpyDeviceToHost));
        LBVH_CHECK(cudaMemcpy(hr.data(), right.get(), (size_t)n_int * 4, cudaMemcpyDeviceToHost));
        LBVH_CHECK(cudaMemcpy(hrange.data(), range.get(), (size_t)n_int * sizeof(int2), cudaMemcpyDeviceToHost));
        auto is_leaf = [&](int c) { return c < 0 || hrange[c].y - hrange[c].x + 1 <= LBVH_LEAF_MAX; };
        if (is_leaf(0)) root_ref = ~((0 << 2) | (int)(n - 1));              // whole scene fits one leaf
        else {
            std::vector<std::pair<int, int>> stack; stack.push_back({ 0, 1 });
            while (!stack.empty()) {
                auto [node, dep] = stack.back(); stack.pop_back();
                if (dep > max_depth) max_depth = dep;
                if (!is_leaf(hl[node])) stack.push_back({ hl[node], dep + 1 });
                if (!is_leaf(hr[node])) stack.push_back({ hr[node], dep + 1 });
            }
        }
    }
    if (host_ref_box && n_int) {                                            // the host SAH build (lbvh_refine_sah mode 2) works from these
        host_ref_box->resize((size_t)n * 6);
        LBVH_CHECK(cudaMemcpy(host_ref_box->data(), leaf_box.get(), (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost));
    }
    if (dev_ref_box && n_int) *dev_ref_box = std::move(leaf_box);           // the GPU builder (lbvh_ploc_rebuild) works from these, on the device

    out->shade = std::move(shade); out->tri_slot = std::move(tri_slot);
    out->nodes = std::move(nodes); out->tris = tris; out->n_nodes = n_nodes_alloc; out->n_tris = n;   // n_tris = BvhTri slots (references)
    out->n_prims = nt;
    out->root = root_ref;
    out->max_depth = max_depth;
    out->bytes = node_bytes + tri_bytes;
    return 0;
}

} // namespace b200pt
