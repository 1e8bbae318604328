// trace_query.cu -- traversal test hook (b200pt_trace_query): caller-given rays through one chosen traversal shape and query kind.
// Every shape runs the __device__ traversal functions the renderer's kernels run, with the template arguments they use (bvh_trace,
// flat_fixed_trace, dyn_round); only the ray source and the result sink differ.  COUNT instantiations add node visits, triangle tests
// and refused pushes; the others are the renderer's own instantiations.
#include "bvh_traverse.cuh"
#include "bvh_dynfetch.cuh"
#include "kernels.h"
#include <algorithm>

namespace b200pt {

namespace {

constexpr int THREADS = 256;

template <int KIND>
__device__ __forceinline__ void query_params(const TraceQuery &q, uint32_t i, float &tmin, float &tmax, uint32_t &target, float &tmax_test) {
    tmin = q.tmin[i]; tmax = q.tmax[i];
    target = KIND == TQ_TARGET ? q.target[i] : 0xFFFFFFFFu;
    tmax_test = KIND == TQ_TARGET ? q.tmax_test[i] : -1.0f;
}

__device__ __forceinline__ void put_closest(const DevScene &sc, const TraceQuery &q, uint32_t i, bool hit, float t, float u, float v, uint32_t gid) {
    uint32_t prim = 0xFFFFFFFFu, inst = 0xFFFFFFFFu;
    if (hit) {
        const float4 *tp = reinterpret_cast<const float4 *>(sc.tris) + (size_t)sc.tri_slot[gid] * 3;
        inst = __float_as_uint(tp[1].w); prim = __float_as_uint(tp[2].w);
    }
    q.t[i] = hit ? t : -1.0f; q.prim[i] = prim; q.inst[i] = inst;
    q.uv[2 * i] = hit ? u : 0.0f; q.uv[2 * i + 1] = hit ? v : 0.0f;
}

__device__ __forceinline__ void put_stats(const TraceQuery &q, uint32_t i, const uint32_t cnt[3]) {
    if (q.stats) { q.stats[3 * i] = cnt[0]; q.stats[3 * i + 1] = cnt[1]; q.stats[3 * i + 2] = cnt[2]; }
}

// One ray per thread (k_extend, k_camera's fallback walk, k_connect, the fused k_shade_hit): the BVH2 stack walk, or the flat walk of
// shared-memory scenes when `flat` is set and the scene has one.
template <bool SMEM, int KIND, bool FMA>
__global__ void __launch_bounds__(THREADS) k_trace_query(DevScene sc, TraceQuery q, int max_stack, bool flat) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    BvhView bv;
    if (SMEM) { bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar); if (!flat) bv.n_flat = 0u; }
    else bv = global_bvh(sc);
    constexpr bool ANY = KIND != TQ_CLOSEST, TGT = KIND == TQ_TARGET;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += gridDim.x * blockDim.x) {
        const float3 o = f3(q.org[3 * i], q.org[3 * i + 1], q.org[3 * i + 2]), d = f3(q.dir[3 * i], q.dir[3 * i + 1], q.dir[3 * i + 2]);
        float tmin, tmax, tmax_test; uint32_t target;
        query_params<KIND>(q, i, tmin, tmax, target, tmax_test);
        HitRec h;
        uint32_t cnt[3] = { 0u, 0u, 0u };
        const bool f = q.stats ? bvh_trace<SMEM, ANY, true, TGT, FMA>(bv, o, d, tmin, tmax, h, stack, (int)blockDim.x, max_stack, &cnt[0], &cnt[1], target, tmax_test, &cnt[2])
                               : bvh_trace<SMEM, ANY, false, TGT, FMA>(bv, o, d, tmin, tmax, h, stack, (int)blockDim.x, max_stack, nullptr, nullptr, target, tmax_test);
        if (ANY) q.occluded[i] = f ? 1u : 0u;
        else put_closest(sc, q, i, f, h.t, h.u, h.v, h.gid);
        put_stats(q, i, cnt);
    }
}

// k_camera's fixed-origin flat walk: every ray starts at org[0]; the per-CTA table of the origin-only terms is built as k_camera builds it.
__global__ void __launch_bounds__(THREADS) k_trace_query_fixed(DevScene sc, TraceQuery q) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    __shared__ float4 fixed_tab[4 * FLAT_FIXED_MAX];
    const BvhView bv = stage_bvh_smem(sc, smem, &bar);
    const float3 eye = f3(q.org[0], q.org[1], q.org[2]);
    for (uint32_t s = threadIdx.x; s < bv.n_flat; s += blockDim.x) flat_fixed_entry(bv, s, eye, fixed_tab);
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += gridDim.x * blockDim.x) {
        HitRec h;
        const bool f = flat_fixed_trace(fixed_tab, bv.n_flat, f3(q.dir[3 * i], q.dir[3 * i + 1], q.dir[3 * i + 2]), q.tmin[i], q.tmax[i], h);
        put_closest(sc, q, i, f, h.t, h.u, h.v, h.gid);
        const uint32_t cnt[3] = { 0u, bv.n_flat, 0u };
        put_stats(q, i, cnt);
    }
}

// The dynamic-fetch shapes (k_extend_dyn, k_shadow_dyn): the same stack column with its DONE sentinel, the same overflow array and the same
// while-while round; each warp takes 32 consecutive rays and runs rounds until all of them are finished.
template <bool SMEM, bool WIDE, int KIND, bool FMA>
__global__ void __launch_bounds__(THREADS) k_trace_query_dyn(DevScene sc, TraceQuery q, int max_stack) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    stack[0] = DYN_DONE;
    BvhView bv;
    if (SMEM) bv = stage_bvh_smem(sc, smem + (size_t)(max_stack + 1) * blockDim.x * sizeof(int), &bar);
    else bv = global_bvh(sc);
    const uint32_t s_base = smem_u32(stack), s_step = blockDim.x * 4u, s_limit = s_base + (uint32_t)(max_stack + 1) * s_step;
    int spill[WIDE ? DYN_SPILL : 1];
    const float4 *nodes4 = reinterpret_cast<const float4 *>(sc.nodes4);
    if (WIDE) bv.root = 0;
    constexpr bool ANY = KIND != TQ_CLOSEST;
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < q.n; base += gridDim.x * blockDim.x) {   // warp-uniform
        const uint32_t i = base + lane;
        DynRay r; r.cur = DYN_DONE; r.gid = DYN_NONE; r.t = 0.0f; r.u = 0.0f; r.v = 0.0f; r.s_top = s_base; r.n_spill = 0;
        if (i < q.n) {
            float tmin, tmax, tmax_test; uint32_t target;
            query_params<KIND>(q, i, tmin, tmax, target, tmax_test);
            // k_shadow_dyn: a light ray accepts up to nextafter(tL), a sky ray and k_extend_dyn up to tmax
            if (KIND == TQ_TARGET) tmax_test = tmax_test >= 0.0f ? tmax_test : light_tmax_test(tmax);
            else tmax_test = tmax;
            dyn_init(r, f3(q.org[3 * i], q.org[3 * i + 1], q.org[3 * i + 2]), f3(q.dir[3 * i], q.dir[3 * i + 1], q.dir[3 * i + 2]), tmin, tmax, tmax_test,
                     KIND == TQ_TARGET ? target : DYN_NONE, bv.root, s_base, s_step);
        }
        bool occluded = false;
        uint32_t cnt[3] = { 0u, 0u, 0u };
        uint32_t act = __ballot_sync(0xFFFFFFFFu, r.cur != DYN_DONE);
        while (act) {
            if (q.stats) act = dyn_round<SMEM, ANY, WIDE, FMA, true>(bv, nodes4, r, s_step, s_limit, spill, [&] { occluded = true; }, cnt);
            else act = dyn_round<SMEM, ANY, WIDE, FMA>(bv, nodes4, r, s_step, s_limit, spill, [&] { occluded = true; });
        }
        if (i < q.n) {
            if (ANY) q.occluded[i] = occluded ? 1u : 0u;
            else put_closest(sc, q, i, r.gid != DYN_NONE, r.t, r.u, r.v, r.gid);
            put_stats(q, i, cnt);
        }
    }
}

using QueryKernel = void (*)(DevScene, TraceQuery, int, bool);
using DynKernel = void (*)(DevScene, TraceQuery, int);
template <bool SMEM, int KIND> QueryKernel query_kernel(bool fma) { return fma ? k_trace_query<SMEM, KIND, true> : k_trace_query<SMEM, KIND, false>; }
template <bool SMEM> QueryKernel query_kernel(int kind, bool fma) {
    return kind == TQ_CLOSEST ? query_kernel<SMEM, TQ_CLOSEST>(fma) : kind == TQ_ANY ? query_kernel<SMEM, TQ_ANY>(fma) : query_kernel<SMEM, TQ_TARGET>(fma);
}
template <bool SMEM, bool WIDE, int KIND> DynKernel dyn_kernel(bool fma) { return fma ? k_trace_query_dyn<SMEM, WIDE, KIND, true> : k_trace_query_dyn<SMEM, WIDE, KIND, false>; }
template <bool SMEM, bool WIDE> DynKernel dyn_kernel(int kind, bool fma) {
    return kind == TQ_CLOSEST ? dyn_kernel<SMEM, WIDE, TQ_CLOSEST>(fma) : kind == TQ_ANY ? dyn_kernel<SMEM, WIDE, TQ_ANY>(fma) : dyn_kernel<SMEM, WIDE, TQ_TARGET>(fma);
}

// opts the kernel in to the dynamic shared memory it needs; false when that exceeds the 227 KB per-CTA limit
template <class K> bool fits_smem(K fn, size_t bytes) {
    cudaFuncAttributes a{};
    if (cudaFuncGetAttributes(&a, fn) != cudaSuccess || bytes + a.sharedSizeBytes > 227u * 1024u) return false;
    return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess;
}

} // namespace

int launch_trace_query(const LaunchCfg &lc, const DevScene &sc, int bvh4_depth, int shape, int kind, bool fma, const TraceQuery &q, cudaStream_t st) {
    if (q.n == 0) return 0;
    const bool staged = sc.bvh_bytes > 0 && (sc.bvh_bytes % 16u) == 0;      // the whole BVH can be copied into shared memory
    const int grid = (int)std::min<uint32_t>((q.n + THREADS - 1) / THREADS, 1024u);
    const size_t stack_bytes = (size_t)lc.max_stack * THREADS * sizeof(int);
    switch (shape) {
    case TQ_SHARED: case TQ_GLOBAL: case TQ_FLAT: {
        const bool smem = shape != TQ_GLOBAL;
        if (shape == TQ_FLAT && sc.n_flat == 0u) return TQ_UNSUPPORTED;
        if (smem && !staged) return TQ_UNSUPPORTED;
        const QueryKernel fn = smem ? query_kernel<true>(kind, fma) : query_kernel<false>(kind, fma);
        const size_t bytes = stack_bytes + (smem ? sc.bvh_bytes : 0u);
        if (!fits_smem(fn, bytes)) return TQ_UNSUPPORTED;
        fn<<<grid, THREADS, bytes, st>>>(sc, q, lc.max_stack, shape == TQ_FLAT);
        break;
    }
    case TQ_FIXED_ORIGIN: {
        if (kind != TQ_CLOSEST || sc.n_flat == 0u || sc.n_flat > FLAT_FIXED_MAX || !staged) return TQ_UNSUPPORTED;
        if (!fits_smem(k_trace_query_fixed, sc.bvh_bytes)) return TQ_UNSUPPORTED;
        k_trace_query_fixed<<<grid, THREADS, sc.bvh_bytes, st>>>(sc, q);
        break;
    }
    case TQ_DYN2: {                                                         // k_extend_dyn / k_shadow_dyn over the BVH2, staged as the renderer stages it
        const DynKernel fn = lc.bvh_in_smem ? dyn_kernel<true, false>(kind, fma) : dyn_kernel<false, false>(kind, fma);
        const size_t bytes = (size_t)(lc.max_stack + 1) * THREADS * sizeof(int) + (lc.bvh_in_smem ? sc.bvh_bytes : 0u);
        if (!fits_smem(fn, bytes)) return TQ_UNSUPPORTED;
        fn<<<grid, THREADS, bytes, st>>>(sc, q, lc.max_stack);
        break;
    }
    case TQ_DYN4: case TQ_DYN4_SPILL: {                                     // the BVH4 with the renderer's shared column (B200PT_WIDE_STACK), or a 4-entry one
        if (sc.nodes4 == nullptr) return TQ_UNSUPPORTED;
        const int entries = bvh4_stack_entries(bvh4_depth, shape == TQ_DYN4 ? lc.wide_cap : 4);
        if (entries == 0) return TQ_UNSUPPORTED;
        const DynKernel fn = dyn_kernel<false, true>(kind, fma);
        const size_t bytes = (size_t)(entries + 1) * THREADS * sizeof(int);
        if (!fits_smem(fn, bytes)) return TQ_UNSUPPORTED;
        fn<<<grid, THREADS, bytes, st>>>(sc, q, entries);
        break;
    }
    default: return TQ_UNSUPPORTED;
    }
    return (int)cudaGetLastError();
}

} // namespace b200pt
