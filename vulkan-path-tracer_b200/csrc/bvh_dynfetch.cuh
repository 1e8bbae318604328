// bvh_dynfetch.cuh -- warp-persistent "while-while" traversal with dynamic ray fetch for scenes whose BVH lives in L2/HBM.
//
// Same query semantics as bvh_traverse.cuh (reference: SH/RayGen.slang:90 TraceRay, SH/RTCommon.slang:47-117 ray queries), different
// execution shape.  One-ray-per-thread loops issue with few of their 32 lanes active on secondary rays: (1) a warp waits for its longest ray, (2) lanes in the node branch and lanes in the leaf
// branch serialise each other, (3) in k_connect most lanes hold no shadow request at all (0.44 shadow rays per hit).  Here
//   * a lane that finishes its ray commits the result and takes the next ray from a warp-local pool (refilled from one global
//     counter per bounce, one atomic per `chunk` rays) as soon as fewer than `thresh` lanes of the warp are still traversing
//     (Aila & Laine 2009, "Understanding the efficiency of ray traversal on GPUs": persistent while-while + dynamic fetch);
//   * the warp alternates a node phase (every lane descends until it holds a leaf) and a leaf phase (one triangle per iteration, lanes
//     leave when they pop an inner node), so each phase runs with most lanes enabled;
//   * shadow requests are compacted on the fly into a per-warp ring in shared memory, so lanes only ever hold real rays.
// The stack column of each thread keeps a DONE sentinel in entry 0: popping an empty stack ends the ray without a separate test.
#pragma once
#include "bvh_traverse.cuh"

namespace b200pt {

constexpr int DYN_DONE = (int)0x80000000;          // never a valid leaf reference (~((first<<2)|count-1) with first < 2^29-1)
constexpr uint32_t DYN_NONE = 0xFFFFFFFFu;

struct DynRay {
    float3 o, d, inv, oi;
    float tmin, tmax, tmax_test;                    // accept tmin < t < tmax_test; boxes are clipped against the current best (<= tmax)
    float t, u, v; uint32_t gid;                    // best hit so far (closest-hit) / unused (any-hit)
    uint32_t target;                                // TARGET any-hit: id of the sampled light triangle (see bvh_traverse.cuh), else 0xFFFFFFFF
    int cur; uint32_t s_top;
    int n_spill;                                    // BVH4 only: entries in the per-thread overflow stack (local memory)
};
constexpr int DYN_SPILL = 96;                       // overflow entries behind the shared-memory stack column (BVH4: up to 3 pushes per level)

__device__ __forceinline__ void dyn_init(DynRay &r, float3 o, float3 d, float tmin, float tmax, float tmax_test, uint32_t target,
                                         int root, uint32_t s_base, uint32_t s_step) {
    r.o = o; r.d = d;
    r.inv = f3(slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z));
    r.oi = f3(o.x * r.inv.x, o.y * r.inv.y, o.z * r.inv.z);
    r.tmin = tmin; r.tmax = tmax; r.tmax_test = tmax_test;
    r.t = tmax; r.u = 0.0f; r.v = 0.0f; r.gid = DYN_NONE; r.target = target;
    r.cur = root; r.s_top = s_base + s_step;        // entry 0 holds DYN_DONE
    r.n_spill = 0;
}

__device__ __forceinline__ void dyn_pop(DynRay &r, uint32_t s_step) {
    r.s_top -= s_step;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r.cur) : "r"(r.s_top) : "memory");
}

// COUNT (test hook only): cnt[0] node visits, cnt[1] triangle tests, cnt[2] pushes refused by a full stack (bvh_trace's counters).
template <bool SMEM, bool FMA_SLABS, bool COUNT = false>
__device__ __forceinline__ void dyn_node_step(const BvhView &b, DynRay &r, uint32_t s_step, uint32_t s_limit, uint32_t *cnt = nullptr) {
    if (COUNT) cnt[0]++;
    const float4 *np = b.nodes + (size_t)r.cur * 4;
    const float4 n0 = ld4<SMEM>(np), n1 = ld4<SMEM>(np + 1), n2 = ld4<SMEM>(np + 2), n3 = ld4<SMEM>(np + 3);
    float ax0, ax1, ay0, ay1, az0, az1, bx0, bx1, by0, by1, bz0, bz1;
    if (FMA_SLABS) {
        ax0 = __fmaf_rn(n0.x, r.inv.x, -r.oi.x); ax1 = __fmaf_rn(n0.w, r.inv.x, -r.oi.x);
        ay0 = __fmaf_rn(n0.y, r.inv.y, -r.oi.y); ay1 = __fmaf_rn(n1.x, r.inv.y, -r.oi.y);
        az0 = __fmaf_rn(n0.z, r.inv.z, -r.oi.z); az1 = __fmaf_rn(n1.y, r.inv.z, -r.oi.z);
        bx0 = __fmaf_rn(n1.z, r.inv.x, -r.oi.x); bx1 = __fmaf_rn(n2.y, r.inv.x, -r.oi.x);
        by0 = __fmaf_rn(n1.w, r.inv.y, -r.oi.y); by1 = __fmaf_rn(n2.z, r.inv.y, -r.oi.y);
        bz0 = __fmaf_rn(n2.x, r.inv.z, -r.oi.z); bz1 = __fmaf_rn(n2.w, r.inv.z, -r.oi.z);
    } else {
        ax0 = (n0.x - r.o.x) * r.inv.x; ax1 = (n0.w - r.o.x) * r.inv.x;
        ay0 = (n0.y - r.o.y) * r.inv.y; ay1 = (n1.x - r.o.y) * r.inv.y;
        az0 = (n0.z - r.o.z) * r.inv.z; az1 = (n1.y - r.o.z) * r.inv.z;
        bx0 = (n1.z - r.o.x) * r.inv.x; bx1 = (n2.y - r.o.x) * r.inv.x;
        by0 = (n1.w - r.o.y) * r.inv.y; by1 = (n2.z - r.o.y) * r.inv.y;
        bz0 = (n2.x - r.o.z) * r.inv.z; bz1 = (n2.w - r.o.z) * r.inv.z;
    }
    const float an = fmaxf(fmaxf(fminf(ax0, ax1), fminf(ay0, ay1)), fmaxf(fminf(az0, az1), r.tmin));
    const float af = fminf(fminf(fmaxf(ax0, ax1), fmaxf(ay0, ay1)), fminf(fmaxf(az0, az1), r.t));
    const float bn = fmaxf(fmaxf(fminf(bx0, bx1), fminf(by0, by1)), fmaxf(fminf(bz0, bz1), r.tmin));
    const float bf = fminf(fminf(fmaxf(bx0, bx1), fmaxf(by0, by1)), fminf(fmaxf(bz0, bz1), r.t));
    const bool ha = an <= af, hb = bn <= bf;
    const int c0 = __float_as_int(n3.x), c1 = __float_as_int(n3.y);
    if (ha && hb) {
        const bool a_first = an <= bn;
        const int near_c = a_first ? c0 : c1, far_c = a_first ? c1 : c0;
        if (r.s_top < s_limit) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(r.s_top), "r"(far_c) : "memory"); r.s_top += s_step; }
        else if (COUNT) cnt[2]++;
        r.cur = near_c;
    } else if (ha) {
        r.cur = c0;
    } else if (hb) {
        r.cur = c1;
    } else {
        dyn_pop(r, s_step);
    }
}

// ---- BVH4 (Bvh4Node, device_types.h): one 128-B node = four child boxes = one memory round trip for four slab tests.
// Traversal of a BVH that lives in L2 is bound by the latency of the dependent node fetches (ncu: long-scoreboard stalls, 50 % issue
// utilisation on BreakfastRoom), so halving the number of round trips per ray matters more than the instructions per step.
// Hit children are ordered front to back with a 5-exchange sorting network on packed keys (entry distance, 2 low mantissa bits
// replaced by the slot number); the nearest is entered, the others are pushed far-to-near.  The shared-memory column holds the usual
// case, deeper stacks overflow to a per-thread local-memory array, so no push is ever dropped.
template <bool COUNT = false>
__device__ __forceinline__ void dyn_push4(DynRay &r, int v, uint32_t s_step, uint32_t s_limit, int *spill, uint32_t *cnt = nullptr) {
    if (r.s_top < s_limit) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(r.s_top), "r"(v) : "memory"); r.s_top += s_step; }
    else if (r.n_spill < DYN_SPILL) spill[r.n_spill++] = v;
    else if (COUNT) cnt[2]++;
}
__device__ __forceinline__ void dyn_pop4(DynRay &r, uint32_t s_step, const int *spill) {
    if (r.n_spill > 0) r.cur = spill[--r.n_spill];
    else dyn_pop(r, s_step);
}
template <bool FMA_SLABS>
__device__ __forceinline__ uint32_t dyn_child_key(const DynRay &r, float lx, float ly, float lz, float hx, float hy, float hz, uint32_t k) {
    float x0, x1, y0, y1, z0, z1;
    if (FMA_SLABS) {
        x0 = __fmaf_rn(lx, r.inv.x, -r.oi.x); x1 = __fmaf_rn(hx, r.inv.x, -r.oi.x);
        y0 = __fmaf_rn(ly, r.inv.y, -r.oi.y); y1 = __fmaf_rn(hy, r.inv.y, -r.oi.y);
        z0 = __fmaf_rn(lz, r.inv.z, -r.oi.z); z1 = __fmaf_rn(hz, r.inv.z, -r.oi.z);
    } else {
        x0 = (lx - r.o.x) * r.inv.x; x1 = (hx - r.o.x) * r.inv.x;
        y0 = (ly - r.o.y) * r.inv.y; y1 = (hy - r.o.y) * r.inv.y;
        z0 = (lz - r.o.z) * r.inv.z; z1 = (hz - r.o.z) * r.inv.z;
    }
    const float tn = fmaxf(fmaxf(fminf(x0, x1), fminf(y0, y1)), fmaxf(fminf(z0, z1), r.tmin));
    const float tf = fminf(fminf(fmaxf(x0, x1), fmaxf(y0, y1)), fminf(fmaxf(z0, z1), r.t));
    return (tn <= tf) ? ((__float_as_uint(tn) & 0xFFFFFFFCu) | k) : 0xFFFFFFFFu;   // tn >= tmin > 0: the bit pattern orders like the value
}
__device__ __forceinline__ int dyn_sel4(float4 ch, uint32_t key) {
    const uint32_t k = key & 3u;
    return __float_as_int(k == 0u ? ch.x : (k == 1u ? ch.y : (k == 2u ? ch.z : ch.w)));
}
template <bool FMA_SLABS, bool COUNT = false>
__device__ __forceinline__ void dyn_node4_step(const float4 *nodes4, DynRay &r, uint32_t s_step, uint32_t s_limit, int *spill, uint32_t *cnt = nullptr) {
    if (COUNT) cnt[0]++;
    const float4 *np = nodes4 + (size_t)r.cur * 8;
    const float4 LX = __ldg(np), LY = __ldg(np + 1), LZ = __ldg(np + 2), HX = __ldg(np + 3), HY = __ldg(np + 4), HZ = __ldg(np + 5), CH = __ldg(np + 6);
    uint32_t k0 = dyn_child_key<FMA_SLABS>(r, LX.x, LY.x, LZ.x, HX.x, HY.x, HZ.x, 0u);
    uint32_t k1 = dyn_child_key<FMA_SLABS>(r, LX.y, LY.y, LZ.y, HX.y, HY.y, HZ.y, 1u);
    uint32_t k2 = dyn_child_key<FMA_SLABS>(r, LX.z, LY.z, LZ.z, HX.z, HY.z, HZ.z, 2u);
    uint32_t k3 = dyn_child_key<FMA_SLABS>(r, LX.w, LY.w, LZ.w, HX.w, HY.w, HZ.w, 3u);
    uint32_t a, b;
    a = min(k0, k1); b = max(k0, k1); k0 = a; k1 = b;
    a = min(k2, k3); b = max(k2, k3); k2 = a; k3 = b;
    a = min(k0, k2); b = max(k0, k2); k0 = a; k2 = b;
    a = min(k1, k3); b = max(k1, k3); k1 = a; k3 = b;
    a = min(k1, k2); b = max(k1, k2); k1 = a; k2 = b;
    if (k0 == 0xFFFFFFFFu) { dyn_pop4(r, s_step, spill); return; }
    r.cur = dyn_sel4(CH, k0);
    if (k1 != 0xFFFFFFFFu) {
        if (k3 != 0xFFFFFFFFu) dyn_push4<COUNT>(r, dyn_sel4(CH, k3), s_step, s_limit, spill, cnt);
        if (k2 != 0xFFFFFFFFu) dyn_push4<COUNT>(r, dyn_sel4(CH, k2), s_step, s_limit, spill, cnt);
        dyn_push4<COUNT>(r, dyn_sel4(CH, k1), s_step, s_limit, spill, cnt);
    }
}

// One triangle of the current leaf.  Returns true when an ANYHIT ray found its occluder (the ray is finished: cur = DYN_DONE).
template <bool SMEM, bool ANYHIT, bool WIDE = false, bool COUNT = false>
__device__ __forceinline__ bool dyn_leaf_step(const BvhView &b, DynRay &r, uint32_t s_step, const int *spill = nullptr, uint32_t *cnt = nullptr) {
    if (COUNT) cnt[1]++;
    const uint32_t ref = (uint32_t)(~r.cur);
    const uint32_t slot = ref >> 2, rest = ref & 3u;
    const float4 *tp = b.tris + (size_t)slot * 3;
    const float4 ta = ld4<SMEM>(tp), tb = ld4<SMEM>(tp + 1), tc = ld4<SMEM>(tp + 2);
    float t, u, v;
    if (tri_test<!ANYHIT>(f3(ta), f3(tb), f3(tc), r.o, r.d, r.tmin, r.tmax_test, t, u, v)) {
        const uint32_t gid = __float_as_uint(ta.w);
        if (ANYHIT) {
            if (t < r.tmax || gid < r.target) { r.cur = DYN_DONE; return true; }
        } else if (t < r.t || (t == r.t && gid < r.gid)) {
            r.t = t; r.u = u; r.v = v; r.gid = gid;
        }
    }
    if (rest == 0u) { if (WIDE) dyn_pop4(r, s_step, spill); else dyn_pop(r, s_step); }
    else r.cur = (int)~(((slot + 1u) << 2) | (rest - 1u));
    return false;
}

// One round of the while-while loop for every lane of the warp: the node phase (each lane descends until it holds a leaf or is done), then
// the leaf phase (one triangle per iteration until the lane pops an inner node or finishes).  on_occluded() runs in the lane whose ANYHIT ray
// just found its occluder.  Returns the ballot of the lanes still traversing.  Shared by k_extend_dyn, k_shadow_dyn and the traversal test
// hook (trace_query.cu).
template <bool SMEM, bool ANYHIT, bool WIDE, bool FMA_SLABS, bool COUNT = false, class OnOccluded>
__device__ __forceinline__ uint32_t dyn_round(const BvhView &b, const float4 *nodes4, DynRay &r, uint32_t s_step, uint32_t s_limit, int *spill,
                                          OnOccluded &&on_occluded, uint32_t *cnt = nullptr) {
    if (WIDE) { while (r.cur >= 0) dyn_node4_step<FMA_SLABS, COUNT>(nodes4, r, s_step, s_limit, spill, cnt); }
    else { while (r.cur >= 0) dyn_node_step<SMEM, FMA_SLABS, COUNT>(b, r, s_step, s_limit, cnt); }
    __syncwarp();
    while (r.cur < 0 && r.cur != DYN_DONE) {
        if (dyn_leaf_step<SMEM, ANYHIT, WIDE, COUNT>(b, r, s_step, spill, cnt)) on_occluded();
    }
    return __ballot_sync(0xFFFFFFFFu, r.cur != DYN_DONE);
}

// Warp-local pool of consecutive work items, refilled from a global counter.  All members are warp-uniform.
struct DynPool {
    uint32_t next, end, chunk, n;
    bool drained;
    __device__ __forceinline__ void init(uint32_t n_items, uint32_t total_warps) {
        next = 0; end = 0; n = n_items; drained = (n_items == 0);
        uint32_t c = (n_items / (total_warps * 4u)) & ~31u;
        chunk = c < 32u ? 32u : (c > 256u ? 256u : c);
    }
    // Hands `cnt` consecutive items to the lanes whose bit is set in `need` (lane rank order); returns this lane's item or DYN_NONE.
    __device__ __forceinline__ uint32_t take(uint32_t need, uint32_t lane, uint32_t *counter) {
        const uint32_t cnt = (uint32_t)__popc(need), rank = (uint32_t)__popc(need & ((1u << lane) - 1u));
        const bool mine = (need >> lane) & 1u;
        const uint32_t avail = end - next;
        uint32_t idx = DYN_NONE;
        if (avail < cnt && !drained) {
            uint32_t nb = 0;
            if (lane == 0) nb = atomicAdd(counter, chunk);
            nb = __shfl_sync(0xFFFFFFFFu, nb, 0);
            if (mine) idx = rank < avail ? next + rank : nb + (rank - avail);
            next = nb + (cnt - avail); end = nb + chunk;
            if (end >= n) { end = n; drained = true; if (next > end) next = end; }
        } else {
            if (mine && rank < avail) idx = next + rank;
            next += cnt < avail ? cnt : avail;
        }
        return (idx < n) ? idx : DYN_NONE;
    }
    __device__ __forceinline__ bool empty() const { return drained && next >= end; }
};

} // namespace b200pt
