// bvh_build_rules.cuh -- the arithmetic that decides a built tree, shared by the device builders (lbvh.cu, ploc.cu) and their host
// restatements (bvh2_ploc_build_host, bvh4_collapse_host).  Every operation is explicitly rounded on the device and plain on the host (nvcc's
// host code is not contracted), so both sides compute the same bits: a GPU tree can be checked node for node against the CPU one.
#pragma once
#include <cmath>
#include <cstdint>
#include "device_types.h"

#ifndef LBVH_LEAF_MAX
#define LBVH_LEAF_MAX 4
#endif

namespace b200pt {

#ifdef __CUDA_ARCH__
#define BR_FADD(a, b) __fadd_rn(a, b)
#define BR_FSUB(a, b) __fsub_rn(a, b)
#define BR_FMUL(a, b) __fmul_rn(a, b)
#define BR_FMA(a, b, c) __fmaf_rn(a, b, c)
#define BR_DADD(a, b) __dadd_rn(a, b)
#define BR_DSUB(a, b) __dsub_rn(a, b)
#define BR_DMUL(a, b) __dmul_rn(a, b)
#else
#define BR_FADD(a, b) ((a) + (b))
#define BR_FSUB(a, b) ((a) - (b))
#define BR_FMUL(a, b) ((a) * (b))
#define BR_FMA(a, b, c) std::fmaf(a, b, c)
#define BR_DADD(a, b) ((a) + (b))
#define BR_DSUB(a, b) ((a) - (b))
#define BR_DMUL(a, b) ((a) * (b))
#endif

// Absolute child-box pad of a scene whose boxes lie inside `box` (lo xyz, hi xyz): 2e-6 x its largest |coordinate|.  The FMA slab test of
// bvh_trace perturbs a plane by <= 6e-8 x |ray origin|, so this keeps it conservative for origins within ~16 scene extents.
__host__ __device__ __forceinline__ float bvh_scene_pad(const float *box) {
    float ext = 0.0f;
    for (int k = 0; k < 6; k++) ext = fmaxf(ext, fabsf(box[k]));
    return BR_FMA(2e-6f, ext, 1e-30f);
}
// A child box as the nodes store it: the unpadded box grown by 4e-7 x its largest |coordinate| on each axis, plus the scene pad.
__host__ __device__ __forceinline__ void bvh_pad_child(const float *box, float pabs, float *lo, float *hi) {
    for (int k = 0; k < 3; k++) {
        const float p = BR_FMA(4e-7f, fmaxf(fabsf(box[k]), fabsf(box[3 + k])), pabs);
        lo[k] = BR_FSUB(box[k], p); hi[k] = BR_FADD(box[3 + k], p);
    }
}

// PLOC distance of two clusters: half the surface area of the union of their boxes.  A NaN (an infinite extent times a zero one) counts as
// +inf, so every cluster still finds a neighbour and every clustering step merges at least one pair.
__host__ __device__ __forceinline__ float ploc_union_area(const float *a, const float *b) {
    const float dx = BR_FSUB(fmaxf(a[3], b[3]), fminf(a[0], b[0]));
    const float dy = BR_FSUB(fmaxf(a[4], b[4]), fminf(a[1], b[1]));
    const float dz = BR_FSUB(fmaxf(a[5], b[5]), fminf(a[2], b[2]));
    const float s = BR_FADD(BR_FADD(BR_FMUL(dx, dy), BR_FMUL(dy, dz)), BR_FMUL(dz, dx));
    return s == s ? s : INFINITY;
}
__host__ __device__ __forceinline__ double bvh_half_area_d(const float *box) {
    const double dx = BR_DSUB((double)box[3], (double)box[0]), dy = BR_DSUB((double)box[4], (double)box[1]), dz = BR_DSUB((double)box[5], (double)box[2]);
    return BR_DADD(BR_DADD(BR_DMUL(dx, dy), BR_DMUL(dy, dz)), BR_DMUL(dz, dx));
}
// Leaf rule of bvh2_sah_build_host's FormLeaves with a node visit priced as one triangle test: a node of cnt <= LBVH_LEAF_MAX references
// (children l, r) is one leaf when testing its references costs no more than visiting it and splitting, cnt x A <= A + A_l cnt_l + A_r cnt_r.
__host__ __device__ __forceinline__ bool ploc_leaf_ok(uint32_t cnt, const float *box, const float *bl, uint32_t cl, const float *br, uint32_t cr) {
    if (cnt == 1) return true;
    if (cnt > (uint32_t)LBVH_LEAF_MAX) return false;
    const double a = bvh_half_area_d(box);
    return BR_DMUL((double)cnt, a) <= BR_DADD(a, BR_DADD(BR_DMUL(bvh_half_area_d(bl), (double)cl), BR_DMUL(bvh_half_area_d(br), (double)cr)));
}

// ---- PLOC (parallel locally-ordered clustering, Meister & Bittner 2018): ploc.cu's kernels and bvh2_ploc_build_host run these ----
// Node ids: references 0 .. n-1 (their Morton slots), inner nodes n .. 2n-2 in the order they are created; child[2 (id - n) + side].
// Search radius in clusters on either side (DESIGN.md section 13: R = 8 / 16 / 32 measured on the fixtures' references).  A compile-time
// constant; the Makefile's EXTRA=-DPLOC_RADIUS=.. builds A/B variants.
#ifndef PLOC_RADIUS
#define PLOC_RADIUS 16u
#endif
struct PlocMeta {       // per node: references below it, output inner nodes and inner-node depth of its subtree, whether it qualifies as a leaf
    uint32_t cnt, sub, dep, leaf;
};
// Position (in the cluster list cl[0, m)) of the nearest neighbour of cluster i: smallest union area, the lower position on ties.
__host__ __device__ __forceinline__ uint32_t ploc_nearest(const uint32_t *cl, uint32_t m, uint32_t i, const float *box) {
    const float *a = box + (size_t)cl[i] * 6;
    const uint32_t lo = i > PLOC_RADIUS ? i - PLOC_RADIUS : 0u, hi = i + PLOC_RADIUS < m ? i + PLOC_RADIUS : m - 1;
    uint32_t best = i; float best_d = 0.0f;
    for (uint32_t j = lo; j <= hi; j++) {
        if (j == i) continue;
        const float d = ploc_union_area(a, box + (size_t)cl[j] * 6);
        if (best == i || d < best_d) { best_d = d; best = j; }
    }
    return best;
}
// Inner node id = (left a, right b): its unpadded box, counts and leaf decision.  sub / dep assume no ancestor becomes a leaf: a qualifying
// node has sub = dep = 0 (it and everything below it is one leaf); the root's sub and dep are the output's node count and depth.
__host__ __device__ __forceinline__ void ploc_merge(uint32_t id, uint32_t a, uint32_t b, uint32_t n, float *box, PlocMeta *meta, uint32_t *child) {
    const float *ba = box + (size_t)a * 6, *bb = box + (size_t)b * 6; float *o = box + (size_t)id * 6;
    for (int k = 0; k < 3; k++) { o[k] = fminf(ba[k], bb[k]); o[3 + k] = fmaxf(ba[3 + k], bb[3 + k]); }
    const PlocMeta ma = meta[a], mb = meta[b];
    PlocMeta r;
    r.cnt = ma.cnt + mb.cnt;
    r.leaf = ploc_leaf_ok(r.cnt, o, ba, ma.cnt, bb, mb.cnt) ? 1u : 0u;
    r.sub = r.leaf ? 0u : 1u + ma.sub + mb.sub;
    r.dep = r.leaf ? 0u : 1u + (ma.dep > mb.dep ? ma.dep : mb.dep);
    meta[id] = r;
    child[2 * (size_t)(id - n)] = a; child[2 * (size_t)(id - n) + 1] = b;
}
// Writes inner node x, which the depth-first layout (left first, root 0) puts at out[idx] with its references from slot `first` on.
// A qualifying child becomes a leaf reference ~(first << 2 | count - 1) and its references (left first) go to perm[first ..]; an inner child
// gets kid_idx / kid_first (kid_idx = UINT32_MAX for a leaf).
__host__ __device__ __forceinline__ void ploc_emit(uint32_t x, uint32_t idx, uint32_t first, uint32_t n, const float *box, const PlocMeta *meta,
                                                   const uint32_t *child, float pabs, BvhNode *out, uint32_t *perm, uint32_t kid_idx[2], uint32_t kid_first[2]) {
    BvhNode nd;
    const uint32_t l = child[2 * (size_t)(x - n)], r = child[2 * (size_t)(x - n) + 1];
    bvh_pad_child(box + (size_t)l * 6, pabs, nd.lo0, nd.hi0);
    bvh_pad_child(box + (size_t)r * 6, pabs, nd.lo1, nd.hi1);
    for (int s = 0; s < 2; s++) {
        const uint32_t c = s ? r : l, f = first + (s ? meta[l].cnt : 0u);
        int32_t ref;
        if (meta[c].leaf) {
            ref = ~(int32_t)((f << 2) | (meta[c].cnt - 1u));
            uint32_t stack[LBVH_LEAF_MAX], sp = 0, k = f;
            stack[sp++] = c;
            while (sp) {
                const uint32_t y = stack[--sp];
                if (y < n) { perm[k++] = y; continue; }
                stack[sp++] = child[2 * (size_t)(y - n) + 1]; stack[sp++] = child[2 * (size_t)(y - n)];
            }
            kid_idx[s] = 0xFFFFFFFFu;
        } else {
            kid_idx[s] = idx + 1u + (s ? meta[l].sub : 0u);
            ref = (int32_t)kid_idx[s];
        }
        kid_first[s] = f;
        if (s) nd.c1 = ref; else nd.c0 = ref;
    }
    nd._pad[0] = nd._pad[1] = 0;
    out[idx] = nd;
}

// Area the BVH2 -> BVH4 collapse ranks internal children by (half surface area of the padded child box, fp32).
__host__ __device__ __forceinline__ float bvh4_slot_area(const float *lo, const float *hi) {
    const float dx = BR_FSUB(hi[0], lo[0]), dy = BR_FSUB(hi[1], lo[1]), dz = BR_FSUB(hi[2], lo[2]);
    return BR_FADD(BR_FADD(BR_FMUL(dx, dy), BR_FMUL(dy, dz)), BR_FMUL(dz, dx));
}

} // namespace b200pt
