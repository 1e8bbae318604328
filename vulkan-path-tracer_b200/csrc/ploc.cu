// ploc.cu -- the GPU tree builder: PLOC (parallel locally-ordered clustering, Meister & Bittner 2018) over the LBVH's Morton-ordered
// reference boxes, SAH leaf formation, depth-first layout, the slot permutation, and the BVH2 -> BVH4 collapse, all on the device.
//
// Every step that decides the tree is a helper of bvh_build_rules.cuh that bvh2_ploc_build_host (lbvh.cu) runs as well: the device tree
// equals the host restatement bit for bit, and the device collapse equals bvh4_collapse_host byte for byte (lbvh_refit_prepare re-derives the
// refit's BVH4 source map by re-running the host collapse, so a different node order would make every later refit write wrong boxes).
#include "kernels.h"
#include "bvh_build_rules.cuh"
#include <vector>
#include <cstdio>
#include <cstdlib>

namespace b200pt {

#define PLOC_CHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

// Exclusive scan over the 256 threads of a block (every thread calls it); *total = the block's sum.
__device__ __forceinline__ uint32_t block_scan256(uint32_t v, uint32_t *total) {
    __shared__ uint32_t wsum[8];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= (uint32_t)o) x += y; }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    if (w == 0) {
        uint32_t s = lane < 8 ? wsum[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, s, o); if (lane >= (uint32_t)o) s += y; }
        if (lane < 8) wsum[lane] = s;
    }
    __syncthreads();
    const uint32_t excl = x - v + (w ? wsum[w - 1] : 0u);
    *total = wsum[7];
    __syncthreads();                                                       // wsum is reused by the next call
    return excl;
}
// Exclusive scan of v[0, n) in place by one block; *total = the sum.
__global__ void __launch_bounds__(256) k_scan_excl(uint32_t *__restrict__ v, uint32_t n, uint32_t *__restrict__ total) {
    uint32_t carry = 0;
    for (uint32_t base = 0; base < n; base += 256) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t x = i < n ? v[i] : 0u;
        uint32_t t;
        const uint32_t e = block_scan256(x, &t);
        if (i < n) v[i] = carry + e;
        carry += t;
    }
    if (threadIdx.x == 0) *total = carry;
}

// ---- clustering ----------------------------------------------------------------------------------------------------------------------
__global__ void k_ploc_init(const float *__restrict__ ref_box, uint32_t n, float *__restrict__ box, PlocMeta *__restrict__ meta, uint32_t *__restrict__ cl) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int k = 0; k < 6; k++) box[(size_t)i * 6 + k] = ref_box[(size_t)i * 6 + k];
    meta[i] = PlocMeta{ 1u, 0u, 0u, 1u };
    cl[i] = i;
}
__global__ void k_ploc_nearest(const uint32_t *__restrict__ cl, uint32_t m, const float *__restrict__ box, uint32_t *__restrict__ nn) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) nn[i] = ploc_nearest(cl, m, i, box);
}
// survivor (bit 16) and merge-into-new-node (bit 0) flags of position i
__device__ __forceinline__ uint32_t ploc_flags(const uint32_t *nn, uint32_t m, uint32_t i) {
    if (i >= m) return 0u;
    const uint32_t j = nn[i];
    const bool mutual = nn[j] == i;
    return (mutual && j < i) ? 0u : ((1u << 16) | (mutual ? 1u : 0u));
}
// bcnt[b] = survivors of block b, bcnt[nb + b] = merges of block b
__global__ void __launch_bounds__(256) k_ploc_count(const uint32_t *__restrict__ nn, uint32_t m, uint32_t *__restrict__ bcnt, uint32_t nb) {
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    uint32_t t;
    block_scan256(ploc_flags(nn, m, i), &t);
    if (threadIdx.x == 0) { bcnt[blockIdx.x] = t >> 16; bcnt[nb + blockIdx.x] = t & 0xFFFFu; }
}
// After the scan of bcnt: bcnt[nb] = all survivors, so merge k of the step (in position order) creates node node_base + k.
__global__ void __launch_bounds__(256) k_ploc_merge(const uint32_t *__restrict__ cl, const uint32_t *__restrict__ nn, uint32_t m, const uint32_t *__restrict__ bcnt,
                                                    uint32_t nb, uint32_t node_base, uint32_t n, float *box, PlocMeta *meta, uint32_t *__restrict__ child,
                                                    uint32_t *__restrict__ cl_out) {
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    const uint32_t f = ploc_flags(nn, m, i);
    uint32_t t;
    const uint32_t e = block_scan256(f, &t);
    if (!(f >> 16)) return;
    uint32_t id = cl[i];
    if (f & 1u) {
        const uint32_t nid = node_base + (bcnt[nb + blockIdx.x] - bcnt[nb]) + (e & 0xFFFFu);
        ploc_merge(nid, id, cl[nn[i]], n, box, meta, child);
        id = nid;
    }
    cl_out[bcnt[blockIdx.x] + (e >> 16)] = id;
}

// ---- layout: inner nodes of one clustering step, latest step first (a parent is always created after its children) -------------------
// place[x - n] = (output index, first slot) of inner node x once its parent has placed it, (UINT32_MAX, 0) while it is below a leaf.
__global__ void k_ploc_emit(uint32_t first_id, uint32_t count, uint32_t n, uint32_t root, const float *__restrict__ box, const PlocMeta *__restrict__ meta,
                            const uint32_t *__restrict__ child, uint2 *__restrict__ place, BvhNode *__restrict__ out, uint32_t *__restrict__ perm) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint32_t x = first_id + i;
    const uint2 p = place[x - n];
    if (p.x == 0xFFFFFFFFu) return;
    const float pabs = bvh_scene_pad(box + (size_t)root * 6);
    uint32_t kid_idx[2], kid_first[2];
    ploc_emit(x, p.x, p.y, n, box, meta, child, pabs, out, perm, kid_idx, kid_first);
    for (int s = 0; s < 2; s++) if (kid_idx[s] != 0xFFFFFFFFu) place[child[2 * (size_t)(x - n) + s] - n] = make_uint2(kid_idx[s], kid_first[s]);
}

int ploc_build(const float *d_ref_box, uint32_t n, BvhNode *d_out, uint32_t *d_perm, uint32_t *n_out, int *depth, uint32_t *h_small, cudaStream_t st) {
    *n_out = 0; *depth = 0;
    if (n <= (uint32_t)LBVH_LEAF_MAX || n >= (1u << 28)) return 0;
    const uint32_t n_all = 2 * n - 1, nb = (n + 255) / 256;
    DevPtr<float> box; DevPtr<PlocMeta> meta; DevPtr<uint32_t> child, cl, nn, bcnt; DevPtr<uint2> place;
    PLOC_CHECK(alloc(box, (size_t)n_all * 6 * sizeof(float)));
    PLOC_CHECK(alloc(meta, (size_t)n_all * sizeof(PlocMeta)));
    PLOC_CHECK(alloc(child, (size_t)(n - 1) * 2 * 4));
    PLOC_CHECK(alloc(cl, (size_t)n * 2 * 4));
    PLOC_CHECK(alloc(nn, (size_t)n * 4));
    PLOC_CHECK(alloc(bcnt, ((size_t)2 * nb + 1) * 4));
    PLOC_CHECK(alloc(place, (size_t)(n - 1) * sizeof(uint2)));
    k_ploc_init<<<nb, 256, 0, st>>>(d_ref_box, n, box.get(), meta.get(), cl.get());
    std::vector<uint32_t> step_m{ n };                                        // clusters at the start of each step
    uint32_t *cur = cl.get(), *nxt = cl.get() + n, m = n;
    while (m > 1) {
        const uint32_t mb = (m + 255) / 256;
        k_ploc_nearest<<<mb, 256, 0, st>>>(cur, m, box.get(), nn.get());
        k_ploc_count<<<mb, 256, 0, st>>>(nn.get(), m, bcnt.get(), mb);
        k_scan_excl<<<1, 256, 0, st>>>(bcnt.get(), 2 * mb, bcnt.get() + 2 * mb);
        k_ploc_merge<<<mb, 256, 0, st>>>(cur, nn.get(), m, bcnt.get(), mb, n + (n - m), n, box.get(), meta.get(), child.get(), nxt);
        PLOC_CHECK(cudaMemcpyAsync(h_small, bcnt.get() + mb, 4, cudaMemcpyDeviceToHost, st));
        PLOC_CHECK(cudaStreamSynchronize(st));
        if (h_small[0] >= m) return (int)cudaErrorUnknown;                     // every step merges at least one pair (ploc_union_area)
        m = h_small[0]; step_m.push_back(m);
        std::swap(cur, nxt);
    }
    const uint32_t root = n_all - 1;
    PLOC_CHECK(cudaMemcpyAsync(h_small, meta.get() + root, sizeof(PlocMeta), cudaMemcpyDeviceToHost, st));
    PLOC_CHECK(cudaMemsetAsync(place.get(), 0xFF, (size_t)(n - 1) * sizeof(uint2), st));
    const uint2 root_place = make_uint2(0u, 0u);
    PLOC_CHECK(cudaMemcpyAsync(place.get() + (root - n), &root_place, sizeof root_place, cudaMemcpyHostToDevice, st));
    for (size_t s = step_m.size() - 1; s-- > 0;) {                           // step s created nodes [n + (n - m_s), n + (n - m_{s+1}))
        const uint32_t first = n + (n - step_m[s]), count = step_m[s] - step_m[s + 1];
        k_ploc_emit<<<(count + 255) / 256, 256, 0, st>>>(first, count, n, root, box.get(), meta.get(), child.get(), place.get(), d_out, d_perm);
    }
    PLOC_CHECK(cudaGetLastError());
    PLOC_CHECK(cudaStreamSynchronize(st));
    *n_out = h_small[1]; *depth = (int)h_small[2];                            // PlocMeta {cnt, sub, dep, leaf} of the root
    return 0;
}

// ---- slot permutation -----------------------------------------------------------------------------------------------------------------
__global__ void k_permute_tris(const BvhTri *__restrict__ src, const uint32_t *__restrict__ perm, uint32_t n, BvhTri *__restrict__ dst, uint32_t *__restrict__ tri_slot) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const BvhTri t = src[perm[i]];
    dst[i] = t;
    atomicMax(&tri_slot[__float_as_uint(t.a.w)], i);                       // the highest of a triangle's slots: deterministic
}

int lbvh_ploc_rebuild(LbvhResult *r, DevPtr<float> ref_box, uint32_t *h_small, cudaStream_t st) {
    const uint32_t n = r->n_tris;
    if (!r->nodes || r->root < 0 || n <= (uint32_t)LBVH_LEAF_MAX || n - 1 > r->n_nodes) return 0;
    DevPtr<BvhNode> nodes; DevPtr<uint32_t> perm; DevPtr<BvhTri> tris;
    PLOC_CHECK(alloc(nodes, (size_t)(n - 1) * sizeof(BvhNode)));
    PLOC_CHECK(alloc(perm, (size_t)n * 4));
    uint32_t n_out = 0; int depth = 0;
    const int e = ploc_build(ref_box.get(), n, nodes.get(), perm.get(), &n_out, &depth, h_small, st);
    if (e != 0) return e;
    // a tree of detail nested around a point can be far deeper than the LBVH: keep the shallower one rather than make every traversal
    // kernel carry a deeper stack (lbvh_refine_sah's rule)
    const bool depth_ok = depth + 2 <= BVH_STACK_MAX || depth <= r->max_depth;
    if (getenv("B200PT_DEBUG"))
        fprintf(stderr, "[b200pt] GPU PLOC build: %u nodes, depth %d (LBVH %d)%s\n", n_out, depth, r->max_depth, depth_ok ? "" : ": too deep, LBVH kept");
    if (n_out == 0 || !depth_ok) return 0;
    PLOC_CHECK(alloc(tris, (size_t)n * sizeof(BvhTri)));
    PLOC_CHECK(cudaMemcpyAsync(tris.get(), r->tris, (size_t)n * sizeof(BvhTri), cudaMemcpyDeviceToDevice, st));
    PLOC_CHECK(cudaMemsetAsync(r->tri_slot.get(), 0, (size_t)r->n_prims * 4, st));
    k_permute_tris<<<(n + 255) / 256, 256, 0, st>>>(tris.get(), perm.get(), n, r->tris, r->tri_slot.get());
    PLOC_CHECK(cudaMemcpyAsync(r->nodes.get(), nodes.get(), (size_t)n_out * sizeof(BvhNode), cudaMemcpyDeviceToDevice, st));
    PLOC_CHECK(cudaGetLastError());
    PLOC_CHECK(cudaStreamSynchronize(st));
    r->root = 0; r->max_depth = depth;
    return 0;
}

// ---- BVH2 -> BVH4, level by level ------------------------------------------------------------------------------------------------------
// The slots of BVH4 node `n2` exactly as bvh4_collapse_host fills them: start from the two children, keep replacing the internal child of
// largest bvh4_slot_area (the first on ties) by its two children until four slots are filled or only leaves remain.
struct C4Slot { int32_t child, src; };
__device__ __forceinline__ int c4_slots(const BvhNode *__restrict__ nodes2, int32_t n2, C4Slot sl[4]) {
    sl[0] = { nodes2[n2].c0, n2 * 2 }; sl[1] = { nodes2[n2].c1, n2 * 2 + 1 };
    int ns = 2;
    while (ns < 4) {
        int best = -1; float best_a = -1.0f;
        for (int k = 0; k < ns; k++) {
            if (sl[k].child < 0) continue;
            const BvhNode &N = nodes2[sl[k].src >> 1];
            const float a = (sl[k].src & 1) ? bvh4_slot_area(N.lo1, N.hi1) : bvh4_slot_area(N.lo0, N.hi0);
            if (a > best_a) { best_a = a; best = k; }
        }
        if (best < 0) break;
        const int32_t c = sl[best].child;
        sl[best] = { nodes2[c].c0, c * 2 }; sl[ns++] = { nodes2[c].c1, c * 2 + 1 };
    }
    return ns;
}
__device__ __forceinline__ uint32_t c4_internal(const BvhNode *nodes2, const int32_t *q2, uint32_t b, uint32_t e, uint32_t i, C4Slot sl[4], int *ns) {
    *ns = 0;
    if (b + i >= e) return 0u;
    *ns = c4_slots(nodes2, q2[b + i], sl);
    uint32_t c = 0;
    for (int k = 0; k < *ns; k++) c += sl[k].child >= 0 ? 1u : 0u;
    return c;
}
// level [b, e) of the BVH4 (q2: the BVH2 node each BVH4 node takes): bcnt[block] = internal children of the block's nodes
__global__ void __launch_bounds__(256) k_c4_count(const BvhNode *__restrict__ nodes2, const int32_t *__restrict__ q2, uint32_t b, uint32_t e, uint32_t *__restrict__ bcnt) {
    C4Slot sl[4]; int ns;
    uint32_t t;
    block_scan256(c4_internal(nodes2, q2, b, e, blockIdx.x * 256 + threadIdx.x, sl, &ns), &t);
    if (threadIdx.x == 0) bcnt[blockIdx.x] = t;
}
// writes the level's BVH4 nodes; their internal children become BVH4 nodes e + (children of earlier nodes of the level), in slot order
__global__ void __launch_bounds__(256) k_c4_emit(const BvhNode *__restrict__ nodes2, int32_t *__restrict__ q2, uint32_t b, uint32_t e, const uint32_t *__restrict__ bcnt,
                                                 Bvh4Node *__restrict__ out) {
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    C4Slot sl[4]; int ns;
    uint32_t t;
    const uint32_t c = c4_internal(nodes2, q2, b, e, i, sl, &ns);
    uint32_t next = e + bcnt[blockIdx.x] + block_scan256(c, &t);
    if (b + i >= e) return;
    Bvh4Node o;
    for (int k = 0; k < 4; k++) {
        if (k < ns) {
            const BvhNode &N = nodes2[sl[k].src >> 1];
            const float *lo = (sl[k].src & 1) ? N.lo1 : N.lo0, *hi = (sl[k].src & 1) ? N.hi1 : N.hi0;
            o.lox[k] = lo[0]; o.loy[k] = lo[1]; o.loz[k] = lo[2]; o.hix[k] = hi[0]; o.hiy[k] = hi[1]; o.hiz[k] = hi[2];
            if (sl[k].child >= 0) { q2[next] = sl[k].child; o.child[k] = (int32_t)next++; }
            else o.child[k] = sl[k].child;
        } else {
            o.lox[k] = o.loy[k] = o.loz[k] = o.hix[k] = o.hiy[k] = o.hiz[k] = 3.0e38f;
            o.child[k] = BVH4_EMPTY;
        }
        o._pad[k] = 0;
    }
    out[b + i] = o;
}

int bvh4_collapse_device(const BvhNode *d_nodes2, uint32_t n_nodes2, int32_t root2, Bvh4Node *d_out, uint32_t *n4, int *depth4, uint32_t *h_total, cudaStream_t st) {
    *n4 = 0; *depth4 = 0;
    if (root2 < 0 || n_nodes2 == 0) return 0;
    const uint32_t nb_max = (n_nodes2 + 255) / 256;
    DevPtr<int32_t> q2; DevPtr<uint32_t> bcnt;
    PLOC_CHECK(alloc(q2, (size_t)n_nodes2 * 4));
    PLOC_CHECK(alloc(bcnt, ((size_t)nb_max + 1) * 4));
    PLOC_CHECK(cudaMemcpyAsync(q2.get(), &root2, 4, cudaMemcpyHostToDevice, st));
    uint32_t b = 0, e = 1; int levels = 0;
    while (b < e) {
        const uint32_t nb = (e - b + 255) / 256;
        k_c4_count<<<nb, 256, 0, st>>>(d_nodes2, q2.get(), b, e, bcnt.get());
        k_scan_excl<<<1, 256, 0, st>>>(bcnt.get(), nb, bcnt.get() + nb);
        k_c4_emit<<<nb, 256, 0, st>>>(d_nodes2, q2.get(), b, e, bcnt.get(), d_out);
        PLOC_CHECK(cudaMemcpyAsync(h_total, bcnt.get() + nb, 4, cudaMemcpyDeviceToHost, st));
        PLOC_CHECK(cudaStreamSynchronize(st));
        levels++;
        if ((uint64_t)e + h_total[0] > n_nodes2) return (int)cudaErrorInvalidValue;   // every BVH4 node consumes at least one BVH2 node
        b = e; e += h_total[0];
    }
    PLOC_CHECK(cudaGetLastError());
    *n4 = e; *depth4 = levels;
    return 0;
}

int lbvh_build_wide_device(LbvhResult *r, uint32_t *h_small, cudaStream_t st) {
    r->nodes4 = nullptr; r->n_nodes4 = 0; r->depth4 = 0;
    if (!r->nodes || r->root < 0 || r->n_nodes == 0) return 0;
    DevPtr<Bvh4Node> scratch, out;                                         // collapsed into room for n_nodes, kept at the exact size
    uint32_t n4 = 0; int d4 = 0;
    PLOC_CHECK(alloc(scratch, (size_t)r->n_nodes * sizeof(Bvh4Node)));
    const int e = bvh4_collapse_device(r->nodes.get(), r->n_nodes, r->root, scratch.get(), &n4, &d4, h_small, st);
    if (e != 0 || n4 == 0) return e;
    PLOC_CHECK(alloc(out, (size_t)n4 * sizeof(Bvh4Node)));
    PLOC_CHECK(cudaMemcpyAsync(out.get(), scratch.get(), (size_t)n4 * sizeof(Bvh4Node), cudaMemcpyDeviceToDevice, st));
    PLOC_CHECK(cudaStreamSynchronize(st));
    r->nodes4 = std::move(out); r->n_nodes4 = n4; r->depth4 = d4;
    return 0;
}

} // namespace b200pt
