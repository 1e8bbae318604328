// bvh_traverse.cuh -- stack traversal of the 64-B two-child-box BVH2 (closest-hit and any-hit).
// Replaces the driver TLAS/BLAS + RT-core traversal behind TraceRay / RayQuery::Proceed
// (reference: SH/RayGen.slang:90, SH/RTCommon.slang:47-117; semantics SURVEY 8a row A1):
//   no culling, force-opaque, accept tmin < t < tmax, report (instance, primitive, t, barycentrics);
//   exact-t ties resolve to the lowest (instance, primitive) order so results are reproducible.
// The traversal stack lives in shared memory (one column per thread, conflict-free); small scenes have
// the whole node + triangle array staged into shared memory by one TMA bulk copy per CTA.
#pragma once
#include "shading.cuh"

namespace b200pt {

struct BvhView { const float4 *nodes; const float4 *tris; int root; uint32_t n_flat; };   // n_flat != 0: no hierarchy, test slots [0, n_flat) in order (tiny scenes in shared memory)
struct HitRec { float t, u, v; uint32_t slot; uint32_t gid; };   // slot: BvhTri (reference) slot; gid: triangle id in (instance, primitive) order

// ---- TMA 1-D bulk copy global -> shared, completion on an mbarrier (sm_90+) ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}

// Stage nodes+tris (contiguous in HBM, `bytes` multiple of 16) into shared memory.  Called by all threads.
// TMA bulk copies are limited in size per instruction, so the copy is issued in 32 KB pieces by thread 0.
__device__ __forceinline__ BvhView stage_bvh_smem(const DevScene &sc, unsigned char *dst, uint64_t *bar) {
    if (threadIdx.x == 0) { mbar_init(bar, 1); }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t total = sc.bvh_bytes;
        mbar_expect_tx(bar, total);
        const unsigned char *src = reinterpret_cast<const unsigned char *>(sc.nodes);
        for (uint32_t off = 0; off < total; off += 32768u) {
            uint32_t n = min(32768u, total - off);
            tma_bulk_g2s(dst + off, src + off, n, bar);
        }
    }
    mbar_wait(bar, 0);
    BvhView v;
    v.nodes = reinterpret_cast<const float4 *>(dst);
    v.tris = reinterpret_cast<const float4 *>(dst + (size_t)sc.n_nodes * sizeof(BvhNode));
    v.root = sc.root; v.n_flat = sc.n_flat;
    return v;
}
__device__ __forceinline__ BvhView global_bvh(const DevScene &sc) {
    BvhView v; v.nodes = reinterpret_cast<const float4 *>(sc.nodes); v.tris = reinterpret_cast<const float4 *>(sc.tris); v.root = sc.root; v.n_flat = 0u; return v;
}

template <bool SMEM> __device__ __forceinline__ float4 ld4(const float4 *p) {
    if (SMEM) return *p; else return __ldg(p);
}

// Moeller-Trumbore with precomputed edges; the same formula as the oracle's tri_hit().
// The products are written with explicit FMA / multiply intrinsics so that every kernel this is inlined into (k_extend, k_connect,
// k_extend_dyn, k_shadow_dyn, k_trace_query) rounds identically: the traversal shapes are interchangeable bit for bit (tested).
__device__ __forceinline__ float3 cross_fma(float3 a, float3 b) {          // a x b, each component fma(a1, b2, -(a2 * b1))
    return f3(__fmaf_rn(a.y, b.z, -__fmul_rn(a.z, b.y)), __fmaf_rn(a.z, b.x, -__fmul_rn(a.x, b.z)), __fmaf_rn(a.x, b.y, -__fmul_rn(a.y, b.x)));
}
__device__ __forceinline__ float dot_fma(float3 a, float3 b) { return __fmaf_rn(a.z, b.z, __fmaf_rn(a.y, b.y, __fmul_rn(a.x, b.x))); }
// normalize() of the extension-ray direction (SH/RayGen.slang:70) with pinned rounding, shared by k_extend and k_extend_dyn
__device__ __forceinline__ float3 normalize_ray(float3 a) {
#ifdef B200PT_PRECISE
    const float inv = 1.0f / sqrtf(dot_fma(a, a));
#else
    const float inv = rsqrtf(dot_fma(a, a));
#endif
    return f3(__fmul_rn(a.x, inv), __fmul_rn(a.y, inv), __fmul_rn(a.z, inv));
}
// Reciprocal of a ray-direction component for the slab tests.  A component that is exactly 0 (axis-aligned NEE / mirror directions) would give
// inv = inf, and the FMA slab form n*inv - o*inv then evaluates inf - inf = NaN for a box that straddles the origin on that axis: fmaxf/fminf drop
// the NaN and the subtree is culled (a false miss).  |d| < 1e-30 is replaced by copysign(1e-30, d): every plane distance stays finite or a
// correctly signed infinity (|n|, |o| < 3e8), the slab interval is unchanged for all practical purposes; the triangle test keeps the exact d.
__device__ __forceinline__ float slab_rcp(float d) { return 1.0f / (fabsf(d) < 1e-30f ? copysignf(1e-30f, d) : d); }
// EARLY = false (any-hit shadow queries): branch-free.  In those loops some lane of a warp passes the u and v tests for nearly every triangle (ncu, flat Cornell
// walk: 95 % / 77 % of the warps enter the second / third stage), so early-outs saved no warp instructions and cost three branch + reconvergence pairs per test
// (k_connect 20.8 -> 19.0 ms per Cornell step).  EARLY = true (closest-hit queries of coherent extension rays): neighbouring rays fail the same test together and
// the early-outs do skip work (k_extend 13.8 -> 12.7 ms).  Both forms evaluate u, v and t with the SAME operations and roundings: identical results.
// 1 / det is the raw reciprocal approximation (MUFU.RCP, 1 ulp) in the default build -- the same precision class as the 2-ulp division it replaces
// (Makefile: -prec-div=false), without the denormal / overflow rescaling around it; PRECISE=1 keeps the IEEE division.
__device__ __forceinline__ float det_rcp(float det) {
#ifdef B200PT_PRECISE
    return 1.0f / det;
#else
    return __fdividef(1.0f, det);
#endif
}
template <bool EARLY = false>
__device__ __forceinline__ bool tri_test(float3 v0, float3 e1, float3 e2, float3 o, float3 d, float tmin, float tmax, float &t, float &u, float &v) {
    const float3 p = cross_fma(d, e2);
    const float det = dot_fma(e1, p);
    if (EARLY && det == 0.0f) return false;
    const float inv = det_rcp(det);
    const float3 tv = f3(__fsub_rn(o.x, v0.x), __fsub_rn(o.y, v0.y), __fsub_rn(o.z, v0.z));
    u = __fmul_rn(dot_fma(tv, p), inv);
    if (EARLY && !(u >= 0.0f && u <= 1.0f)) return false;
    const float3 q = cross_fma(tv, e1);
    v = __fmul_rn(dot_fma(d, q), inv);
    if (EARLY && !(v >= 0.0f && __fadd_rn(u, v) <= 1.0f)) return false;
    t = __fmul_rn(dot_fma(e2, q), inv);
    if (EARLY) return (t > tmin && t < tmax);
    return (det != 0.0f) & (u >= 0.0f) & (u <= 1.0f) & (v >= 0.0f) & (__fadd_rn(u, v) <= 1.0f) & (t > tmin) & (t < tmax);
}

// Acceptance bound of a light-visibility (TARGET) query whose target the ray hits at tL: the next float above tL, so the target's own hit
// and exact ties at tL pass the triangle test and the tie rule decides them.  Shared by bvh_trace, the fused k_shade_hit, k_shadow_dyn
// and the traversal test hook.
__device__ __forceinline__ float light_tmax_test(float tL) { return __uint_as_float(__float_as_uint(tL) + 1u); }

// stack: shared-memory column of this thread, entries at stack[k * stride] (addressed through the shared window: STS/LDS with
// an incrementally maintained address instead of a generic-pointer computation per push).
// Slab test: with FMA_SLABS the plane distances are one FFMA each, t = n*inv - (o*inv) (12 FFMA per node instead of 12 FADD + 12 FMUL).
// That form perturbs a plane by <= 6e-8*|o| (the rounding of o*inv); the node boxes carry an absolute pad of 2e-6 * scene extent
// (lbvh.cu: k_emit), so it is conservative for every origin within ~16 scene extents -- i.e. for all secondary rays, whose origins lie
// on scene surfaces.  Camera rays (origin anywhere) use the subtract-then-multiply form (FMA_SLABS = false).
// TARGET (with ANYHIT): "is anything in front of triangle target_gid, which the ray hits at tmax?"  A triangle occludes when
// t < tmax, or t == tmax and its id is lower than the target's (the tie rule of the closest-hit query); the target itself never does.
// COUNT: node visits, triangle tests and pushes refused by a full stack (a refused push drops a subtree: wrong answers, not a fault).
template <bool SMEM, bool ANYHIT, bool COUNT = false, bool TARGET = false, bool FMA_SLABS = false>
__device__ __forceinline__ bool bvh_trace(const BvhView &b, float3 o, float3 d, float tmin, float tmax, HitRec &h,
                                          int *stack, int stride, int max_stack, uint32_t *n_nodes = nullptr, uint32_t *n_tris = nullptr,
                                          uint32_t target_gid = 0xFFFFFFFFu, float tmax_test_in = -1.0f, uint32_t *n_refused = nullptr) {
    // TARGET: admit t == tmax (tmax > 0).  A caller that serves both NEE queries with one copy of this loop (the fused k_shade_hit) passes the
    // acceptance bound itself: nextafter(tL) for a light ray, tmax for a sky ray (whose target 0xFFFFFFFF makes every t < tmax an occluder).
    const float tmax_test = TARGET ? (tmax_test_in >= 0.0f ? tmax_test_in : light_tmax_test(tmax)) : tmax;
    h.slot = 0xFFFFFFFFu; h.gid = 0xFFFFFFFFu; h.t = tmax; h.u = 0.0f; h.v = 0.0f;
    uint32_t best_gid = 0xFFFFFFFFu;
    bool found = false;
    // one triangle slot; returns true when an ANYHIT query is decided
    auto test_slot = [&](uint32_t slot) -> bool {
        if (COUNT) (*n_tris)++;
        const float4 *tp = b.tris + (size_t)slot * 3;
        const float4 ta = ld4<SMEM>(tp), tb = ld4<SMEM>(tp + 1), tc = ld4<SMEM>(tp + 2);
        float t, u, v;
        if (tri_test<!ANYHIT>(f3(ta), f3(tb), f3(tc), o, d, tmin, tmax_test, t, u, v)) {
            const uint32_t gid = __float_as_uint(ta.w);
            if (TARGET && !(t < tmax || gid < target_gid)) return false;
            if (!found || t < h.t || (t == h.t && gid < best_gid)) {
                found = true; h.t = t; h.u = u; h.v = v; h.slot = slot; h.gid = gid; best_gid = gid;
                if (ANYHIT) return true;
            }
        }
        return false;
    };
    // Flat mode (SMEM only): a scene of a handful of triangles (the 12-triangle Cornell box) is tested slot by slot with no hierarchy -- every
    // lane walks the same slots (shared-memory broadcasts, no stack, no divergence), which costs fewer instructions than the ~4 node steps +
    // ~2.4 triangle tests of the SAH tree at half-empty warps.  Same tests, same tie rule: identical hits.
    if (SMEM && b.n_flat) {
        for (uint32_t slot = 0; slot < b.n_flat; slot++) if (test_slot(slot)) return true;
        if (!found) h.t = -1.0f;
        return found;
    }
    const float3 inv = f3(slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z));
    const float3 oi = f3(o.x * inv.x, o.y * inv.y, o.z * inv.z);
    const uint32_t s_base = smem_u32(stack), s_step = (uint32_t)stride * 4u, s_limit = s_base + (uint32_t)max_stack * s_step;
    uint32_t s_top = s_base;                                               // address of the next free stack entry
    int cur = b.root;
    while (true) {
        if (cur >= 0) {
            if (COUNT) (*n_nodes)++;
            const float4 *np = b.nodes + (size_t)cur * 4;
            const float4 n0 = ld4<SMEM>(np), n1 = ld4<SMEM>(np + 1), n2 = ld4<SMEM>(np + 2), n3 = ld4<SMEM>(np + 3);
            // child 0: lo (n0.x n0.y n0.z) hi (n0.w n1.x n1.y); child 1: lo (n1.z n1.w n2.x) hi (n2.y n2.z n2.w)
            float ax0, ax1, ay0, ay1, az0, az1, bx0, bx1, by0, by1, bz0, bz1;
            if (FMA_SLABS) {
                ax0 = __fmaf_rn(n0.x, inv.x, -oi.x); ax1 = __fmaf_rn(n0.w, inv.x, -oi.x);
                ay0 = __fmaf_rn(n0.y, inv.y, -oi.y); ay1 = __fmaf_rn(n1.x, inv.y, -oi.y);
                az0 = __fmaf_rn(n0.z, inv.z, -oi.z); az1 = __fmaf_rn(n1.y, inv.z, -oi.z);
                bx0 = __fmaf_rn(n1.z, inv.x, -oi.x); bx1 = __fmaf_rn(n2.y, inv.x, -oi.x);
                by0 = __fmaf_rn(n1.w, inv.y, -oi.y); by1 = __fmaf_rn(n2.z, inv.y, -oi.y);
                bz0 = __fmaf_rn(n2.x, inv.z, -oi.z); bz1 = __fmaf_rn(n2.w, inv.z, -oi.z);
            } else {
                ax0 = (n0.x - o.x) * inv.x; ax1 = (n0.w - o.x) * inv.x;
                ay0 = (n0.y - o.y) * inv.y; ay1 = (n1.x - o.y) * inv.y;
                az0 = (n0.z - o.z) * inv.z; az1 = (n1.y - o.z) * inv.z;
                bx0 = (n1.z - o.x) * inv.x; bx1 = (n2.y - o.x) * inv.x;
                by0 = (n1.w - o.y) * inv.y; by1 = (n2.z - o.y) * inv.y;
                bz0 = (n2.x - o.z) * inv.z; bz1 = (n2.w - o.z) * inv.z;
            }
            const float an = fmaxf(fmaxf(fminf(ax0, ax1), fminf(ay0, ay1)), fmaxf(fminf(az0, az1), tmin));
            const float af = fminf(fminf(fmaxf(ax0, ax1), fmaxf(ay0, ay1)), fminf(fmaxf(az0, az1), h.t));
            const float bn = fmaxf(fmaxf(fminf(bx0, bx1), fminf(by0, by1)), fmaxf(fminf(bz0, bz1), tmin));
            const float bf = fminf(fminf(fmaxf(bx0, bx1), fmaxf(by0, by1)), fminf(fmaxf(bz0, bz1), h.t));
            const bool ha = an <= af, hb = bn <= bf;                        // the boxes are padded (k_emit), no slack needed here
            const int c0 = __float_as_int(n3.x), c1 = __float_as_int(n3.y);
            if (ha && hb) {
                const bool a_first = an <= bn;
                const int near_c = a_first ? c0 : c1, far_c = a_first ? c1 : c0;
                if (s_top < s_limit) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(s_top), "r"(far_c) : "memory"); s_top += s_step; }
                else if (COUNT && n_refused) (*n_refused)++;
                cur = near_c;
                continue;
            } else if (ha) { cur = c0; continue; }
            else if (hb) { cur = c1; continue; }
        } else {
            const uint32_t ref = (uint32_t)(~cur);                            // leaf: up to 4 consecutive Morton slots
            const uint32_t first = ref >> 2, count = (ref & 3u) + 1u;
            for (uint32_t q = 0; q < count; q++) if (test_slot(first + q)) return true;
        }
        if (s_top == s_base) break;
        s_top -= s_step;
        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(cur) : "r"(s_top) : "memory");
    }
    if (!found) h.t = -1.0f;
    return found;
}

// Flat closest-hit walk of rays that all start at ONE origin O (pinhole camera rays, k_camera).  The parts of tri_test that depend only on O
// and the triangle -- tv = O - v0, q = tv x e1 and t's numerator e2 . q -- are computed once per CTA into a table; the per-ray rest and the
// tie rule are tri_test<true> / bvh_trace's flat walk operation for operation (all explicitly rounded), so the hits are bit-identical.
// Entry of slot s: [4s] e1 + gid, [4s+1] e2 + e2 . q, [4s+2] tv + q.x, [4s+3] q.y, q.z.
constexpr uint32_t FLAT_FIXED_MAX = 64;                                     // B200PT_FLAT_MAX's upper limit
__device__ __forceinline__ void flat_fixed_entry(const BvhView &b, uint32_t slot, float3 O, float4 *tab) {
    const float4 *tp = b.tris + (size_t)slot * 3;
    const float4 ta = tp[0], tb = tp[1], tc = tp[2];
    const float3 tv = f3(__fsub_rn(O.x, ta.x), __fsub_rn(O.y, ta.y), __fsub_rn(O.z, ta.z));
    const float3 q = cross_fma(tv, f3(tb));
    tab[4 * slot] = make_float4(tb.x, tb.y, tb.z, ta.w);
    tab[4 * slot + 1] = make_float4(tc.x, tc.y, tc.z, dot_fma(f3(tc), q));
    tab[4 * slot + 2] = make_float4(tv.x, tv.y, tv.z, q.x);
    tab[4 * slot + 3] = make_float4(q.y, q.z, 0.0f, 0.0f);
}
__device__ __forceinline__ bool flat_fixed_trace(const float4 *tab, uint32_t n, float3 d, float tmin, float tmax, HitRec &h) {
    h.slot = 0xFFFFFFFFu; h.gid = 0xFFFFFFFFu; h.t = tmax; h.u = 0.0f; h.v = 0.0f;
    uint32_t best_gid = 0xFFFFFFFFu;
    bool found = false;
    for (uint32_t s = 0; s < n; s++) {
        const float4 a = tab[4 * s], b = tab[4 * s + 1], c = tab[4 * s + 2];
        const float3 p = cross_fma(d, f3(b));
        const float det = dot_fma(f3(a), p);
        if (det == 0.0f) continue;
        const float inv = det_rcp(det);
        const float u = __fmul_rn(dot_fma(f3(c), p), inv);
        if (!(u >= 0.0f && u <= 1.0f)) continue;
        const float4 e = tab[4 * s + 3];
        const float v = __fmul_rn(dot_fma(d, f3(c.w, e.x, e.y)), inv);
        if (!(v >= 0.0f && __fadd_rn(u, v) <= 1.0f)) continue;
        const float t = __fmul_rn(b.w, inv);
        if (!(t > tmin && t < tmax)) continue;
        const uint32_t gid = __float_as_uint(a.w);
        if (!found || t < h.t || (t == h.t && gid < best_gid)) { found = true; h.t = t; h.u = u; h.v = v; h.slot = s; h.gid = gid; best_gid = gid; }
    }
    if (!found) h.t = -1.0f;
    return found;
}

} // namespace b200pt
