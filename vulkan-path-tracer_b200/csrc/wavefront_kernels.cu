// wavefront_kernels.cu -- the per-bounce kernels of the wavefront integrator (sm_90a).
//
// The reference runs ONE ray-gen megakernel per frame that loops over bounces and calls TraceRay /
// closest-hit / miss inline (SH/RayGen.slang:9-160).  Here the same estimator is a wavefront:
//
//   k_raygen   camera sample + payload init                    SH/RayGen.slang:12-63
//              (k_camera: the same + the camera rays' k_extend in one kernel, shared-memory scenes without a pre-pass)
//   per bounce:
//     k_extend   closest-hit traversal of the live paths       SH/RayGen.slang:68-72,90 (TraceRay)
//                + sort into the miss queue and one hit queue per MATERIAL CLASS (lobe set)
//     k_shade_miss  miss shading of the miss queue             SH/Miss.slang:8-76
//     k_shade_hit<CLASS>  closest-hit shading of one class's   SH/ClosestHit.slang:20-378
//                   hit queue, emits <=2 NEE shadow requests
//     k_connect  shadow rays, payload.Emitted assembly,        SH/ClosestHit.slang:139,171-176,326-372
//                luminance clamp, throughput, Russian          SH/RayGen.slang:92-113
//                roulette, ballot/prefix-sum compaction
//   scenes whose BVH is staged in shared memory by TMA fuse the shadow queries and the roulette into k_shade_hit<CLASS, ., true> (default).
//   k_resolve  NaN/Inf rejection + running mean                SH/RayGen.slang:116-159
//   (adaptive sampling, no reference equivalent: k_raygen / k_camera over a list of active pixels, k_resolve_adaptive, and
//    k_adaptive_update + k_adaptive_compact at interval boundaries)
//
// Every path owns one sample slot, so radiance accumulation needs no atomics and is deterministic.
// All per-path state is SoA float4 (coalesced 16-B lanes); live paths are kept dense by compaction.
#include "bvh_traverse.cuh"
#include "bvh_dynfetch.cuh"
#include "camera.cuh"
#include "atmosphere.cuh"
#include "kernels.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace b200pt {

// partition helper part_global_row, camera_eye and camera_ray: camera.cuh
// control block (device memory, u32): device_types.h (CTRL_Q)

// ------------------------------------------------------------------------------------------------
// camera_path : camera sample + payload init of path j of a wave (k_raygen, k_camera); returns the camera ray
// ADAPTIVE: the wave holds P = A active pixels per dispatch, entry i of a dispatch traces local pixel active[i] (adaptive sampling).  Only the
// pixel changes: the slot stays j, and the RNG is keyed on the pixel as always, so a pixel's frames are those of the plain renderer.
// flags (kernels.h): WAVE_STORE skips the clear of the sample slot, WAVE_IMPLIED skips the stores of org_pdf, thr_depth and rad_slot (the
// bounce-0 kernels infer them from the camera_implied_* helpers below, which are also what this function writes otherwise).
// ------------------------------------------------------------------------------------------------
constexpr float CAMERA_IMPLIED_PDF = 1.0f;                                  // payload.PDF of a camera path
__device__ __forceinline__ float4 camera_implied_thr_depth(bool inside) {   // throughput 1, Depth 0 (born dead: MAX)
    return make_float4(1.0f, 1.0f, 1.0f, __uint_as_float(inside ? 0u : PT_MAX_DEPTH));
}
__device__ __forceinline__ float4 camera_implied_rad_slot(uint32_t j) {     // no radiance yet, sample slot j
    return make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(j));
}
template <bool ADAPTIVE>
__device__ __forceinline__ void camera_path(const DevConfig &cfg, const DevDispatch *__restrict__ disp, uint32_t P, uint32_t first_sample, uint32_t flags,
                                            const uint32_t *__restrict__ rng_carry, const PathState &ps, float4 *__restrict__ sample_buf,
                                            uint32_t j, float3 &ray_o, float3 &ray_d, const uint32_t *__restrict__ active) {
    const uint32_t S = cfg.ScreenSplitCount;
    const uint32_t LW = (cfg.W + S - 1) / S;
    {
        const uint32_t b = j / P, i = j - b * P;
        const uint32_t p = ADAPTIVE ? __ldg(active + i) : i;
        const DevDispatch dd = disp[b];
        uint32_t x, y;
        if (S == 1) {
            const uint32_t lr = p / cfg.W; x = p - lr * cfg.W;
            y = part_global_row(lr, cfg.rank, cfg.world, cfg.band_rows);
        } else {                                                           // SH/RayGen.slang:17-22
            const uint32_t ly = p / LW, lx = p - ly * LW;
            x = lx * S + dd.ChunkIndex % S; y = ly * S + dd.ChunkIndex / S;
        }
        const bool inside = (x < cfg.W && y < cfg.H);                      // :24-25
        Rng rng;
        if (first_sample) {                                                 // :28 (Q13)
            rng.s = y + cfg.W * x + dd.Seed;
            if (!(flags & WAVE_STORE)) sample_buf[j] = make_float4(0, 0, 0, 0);
        } else rng.s = rng_carry[j];
        float3 origin, direction;
        camera_ray(cfg, x, y, rng, origin, direction);                      // :35-50
        // payload init :52-63.  Pixels outside the image (chunked dispatch overhang) are born dead (Depth = MAX).
        ps.dir_rng[j] = make_float4(direction.x, direction.y, direction.z, __uint_as_float(rng.s));
        if (!(flags & WAVE_IMPLIED)) {
            ps.org_pdf[j] = make_float4(origin.x, origin.y, origin.z, CAMERA_IMPLIED_PDF);
            ps.thr_depth[j] = camera_implied_thr_depth(inside);
            ps.rad_slot[j] = camera_implied_rad_slot(j);
        }
        if (ps.vol_depth) ps.vol_depth[j] = 0u;                             // payload.VolumeDepth = 0 (SH/RayGen.slang:61)
        ray_o = origin; ray_d = direction;
    }
}

// ------------------------------------------------------------------------------------------------
// k_raygen (pipelines without k_camera: volumes / atmosphere pre-pass, BVH outside shared memory, B200PT_CAMERA=0)
// ------------------------------------------------------------------------------------------------
// ADAPTIVE: P = the active count, entry i traces pixel active[i] (camera_path); `active` is unused otherwise.
template <bool ADAPTIVE>
__global__ void __launch_bounds__(256) k_raygen(DevConfig cfg, const DevDispatch *__restrict__ disp, uint32_t n_disp, uint32_t P,
                                                 uint32_t first_sample, uint32_t flags, const uint32_t *__restrict__ rng_carry,
                                                 PathState ps, float4 *__restrict__ sample_buf, uint32_t *__restrict__ ctrl,
                                                 WaveCounters *ctr, const uint32_t *__restrict__ active) {
    const uint32_t n = n_disp * P;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        float3 o, d;
        camera_path<ADAPTIVE>(cfg, disp, P, first_sample, flags, rng_carry, ps, sample_buf, j, o, d, active);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { for (uint32_t w = 0; w < CTRL_WORDS; w++) ctrl[w] = 0; ctrl[0] = n; atomicAdd(&ctr->paths, (unsigned long long)n); }
}

// ------------------------------------------------------------------------------------------------
// queue helpers (device_types.h: Queues, CTRL_Q).  Queue codes: 0 = miss, 1 + c = hit of material class c, Q_NONE = inactive lane.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void ctrl_reset_parity(uint32_t *ctrl, uint32_t q) {   // counters of a bounce with parity q (called by ONE thread, before any writer of that bounce)
    ctrl[q] = 0; ctrl[8u + q] = 0; ctrl[10u + q] = 0;
    #pragma unroll
    for (uint32_t c = 0; c < 1u + MC_COUNT; c++) ctrl[CTRL_Q + 8u * q + c] = 0;
}
// All hit queues of one bounce seen as one list of n entries (k_connect, k_shadow_dyn, k_shade_volume walk every hit whatever its class)
struct HitSpan { uint32_t p1, p2, p3, n; };
__device__ __forceinline__ HitSpan hit_span(const uint32_t *ctrl, uint32_t parity) {
    const uint32_t *c = ctrl + CTRL_Q + 8u * parity + 1u;
    HitSpan h; h.p1 = c[0]; h.p2 = h.p1 + c[1]; h.p3 = h.p2 + c[2]; h.n = h.p3 + c[3];
    return h;
}
__device__ __forceinline__ uint32_t hit_entry(const Queues &q, const HitSpan &h, uint32_t j) {
    const uint32_t c = (uint32_t)(j >= h.p1) + (uint32_t)(j >= h.p2) + (uint32_t)(j >= h.p3);
    const uint32_t base = c == 0u ? 0u : (c == 1u ? h.p1 : (c == 2u ? h.p2 : h.p3));
    return q.hit[(size_t)c * q.cap + (j - base)];
}
__device__ __forceinline__ uint32_t hit_code(const DevScene &sc, uint32_t gid) {   // queue code of a hit on triangle gid
    return 1u + (gid == VOLUME_EVENT ? (uint32_t)MC_GENERAL : (uint32_t)__ldg(sc.tri_class + gid));
}
// Warp-level append of one entry per lane (code Q_NONE = nothing): the lowest lane of every code group reserves room for its group with one
// atomic -- a single atomic instruction with up to five distinct addresses per warp.  Must be called by all 32 lanes.
__device__ __forceinline__ void queue_append(uint32_t code, uint32_t entry, uint32_t *qc, const Queues &q, uint32_t lane) {
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, code);
    const int leader = __ffs((int)peers) - 1;
    uint32_t base = 0;
    if ((int)lane == leader && code != Q_NONE) base = atomicAdd(qc + code, (uint32_t)__popc(peers));
    base = __shfl_sync(0xFFFFFFFFu, base, leader);
    const uint32_t k = base + (uint32_t)__popc(peers & ((1u << lane) - 1u));
    if (code == 0u) q.miss[k] = entry;
    else if (code != Q_NONE) q.hit[(size_t)(code - 1u) * q.cap + k] = entry;
}

// ------------------------------------------------------------------------------------------------
// k_extend : closest hit for every live path; sorts the live list into the miss queue and one hit queue per material class
//            (material-sorted shading: every k_shade_hit<CLASS> warp runs one lobe set, converged)
// ------------------------------------------------------------------------------------------------
// Queue append without block barriers and with few atomics (ncu round 1: returning per-warp atomics on hot addresses were
// 51 % of this kernel's stalls; the block-level scan that replaced them left 2.9 warps/issue parked on __syncthreads).
// A block owns SEGMENTS of K*blockDim consecutive paths (grid-stride over segments); in iteration `it` its warps cover blockDim
// consecutive paths (neighbouring pixels -> shared BVH nodes in L1), each warp traces its K rays without ever waiting for the
// others.  A tally keeps the warp's queue codes of the K iterations, then ONE atomic instruction per warp reserves room in every
// queue for all K iterations.  K adapts to the live count so small waves still fill the GPU.  (k_extend, k_camera)
//
// UniformTally: scenes whose materials all fall into ONE class (and have no volumes) need no per-hit class lookup and only two queues: lane
// `it` keeps the hit / miss ballots of iteration `it`, one atomic instruction reserves room in both (the miss count and the class's hit count
// are not adjacent words, so two lanes issue one 32-bit atomic each in the same instruction).
// Neither tally keeps running totals across the traversals: lanes 0..K-1 hold every iteration's ballots / counts, and the flush sums them.
struct UniformTally {
    uint32_t my_bh = 0u, my_bm = 0u;
    __device__ __forceinline__ void add(uint32_t it, uint32_t lane, bool active, bool hit) {
        const uint32_t bh = __ballot_sync(0xFFFFFFFFu, hit), bm = __ballot_sync(0xFFFFFFFFu, active && !hit);
        if (lane == it) { my_bh = bh; my_bm = bm; }
    }
    // the entry of iteration `it` is path i0 + lane + it * step
    __device__ __forceinline__ void flush(uint32_t K, uint32_t i0, uint32_t step, uint32_t lane, uint32_t *qc, uint32_t cls, const Queues &q) const {
        uint32_t *const q_hit_u = q.hit + (size_t)cls * q.cap;
        const uint32_t lt = (1u << lane) - 1u;
        const uint32_t ch = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)__popc(my_bh)), cm = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)__popc(my_bm));
        uint32_t base = 0u;
        if (lane == 0u && cm) base = atomicAdd(qc, cm);
        else if (lane == 1u && ch) base = atomicAdd(qc + 1u + cls, ch);
        uint32_t om = __shfl_sync(0xFFFFFFFFu, base, 0), oh = __shfl_sync(0xFFFFFFFFu, base, 1);
        uint32_t i = i0 + lane;
        for (uint32_t it = 0; it < K; it++, i += step) {
            const uint32_t bh = __shfl_sync(0xFFFFFFFFu, my_bh, (int)it), bm = __shfl_sync(0xFFFFFFFFu, my_bm, (int)it);
            if ((bh >> lane) & 1u) q_hit_u[oh + __popc(bh & lt)] = i;
            else if ((bm >> lane) & 1u) q.miss[om + __popc(bm & lt)] = i;
            oh += (uint32_t)__popc(bh); om += (uint32_t)__popc(bm);
        }
    }
};
// ClassTally: every lane keeps the queue codes of its K rays (3 bits each), lane `it` keeps the per-queue counts of iteration `it` (6 bits x 5
// queues, one redux), lanes 0..4 reserve room in one queue each.
struct ClassTally {
    uint32_t codes = 0u, my_cnts = 0u;
    __device__ __forceinline__ void skip(uint32_t it) { codes |= Q_NONE << (3u * it); }
    __device__ __forceinline__ void add(uint32_t it, uint32_t lane, uint32_t code) {
        const uint32_t cn = __reduce_add_sync(0xFFFFFFFFu, code != Q_NONE ? 1u << (6u * code) : 0u);
        codes |= code << (3u * it);
        if (lane == it) my_cnts = cn;
    }
    __device__ __forceinline__ void flush(uint32_t K, uint32_t i0, uint32_t step, uint32_t lane, uint32_t *qc, const Queues &q) const {
        const uint32_t lt = (1u << lane) - 1u;
        const uint32_t cn = my_cnts;                                        // totA: queues 0..2, totB: queues 3..4 (10-bit fields, <= 256 each)
        const uint32_t totA = __reduce_add_sync(0xFFFFFFFFu, (cn & 63u) | (((cn >> 6) & 63u) << 10) | (((cn >> 12) & 63u) << 20));
        const uint32_t totB = __reduce_add_sync(0xFFFFFFFFu, ((cn >> 18) & 63u) | (((cn >> 24) & 63u) << 10));
        uint32_t base = 0u;
        {
            const uint32_t mytot = lane < 3u ? (totA >> (10u * lane)) & 1023u : (lane < 5u ? (totB >> (10u * (lane - 3u))) & 1023u : 0u);
            if (mytot) base = atomicAdd(qc + lane, mytot);
        }
        uint32_t runA = 0u, runB = 0u;
        uint32_t i = i0 + lane;
        for (uint32_t it = 0; it < K; it++, i += step) {
            const uint32_t code = (codes >> (3u * it)) & 7u;
            const uint32_t cn = __shfl_sync(0xFFFFFFFFu, my_cnts, (int)it);
            const uint32_t peers = __match_any_sync(0xFFFFFFFFu, code);
            const uint32_t b = __shfl_sync(0xFFFFFFFFu, base, (int)(code < 5u ? code : 0u));
            if (code != Q_NONE) {
                const uint32_t run = code < 3u ? (runA >> (10u * code)) & 1023u : (runB >> (10u * (code - 3u))) & 1023u;
                const uint32_t k = b + run + (uint32_t)__popc(peers & lt);
                if (code == 0u) q.miss[k] = i; else q.hit[(size_t)(code - 1u) * q.cap + k] = i;
            }
            runA += (cn & 63u) | (((cn >> 6) & 63u) << 10) | (((cn >> 12) & 63u) << 20);
            runB += ((cn >> 18) & 63u) | (((cn >> 24) & 63u) << 10);
        }
    }
};

// The shared-memory instantiations of k_extend are held to 80 registers, so that 3 CTAs of 256 threads share an SM: 24 warps hide the flat
// loop's broadcast LDS -> dependent FMA chains, where 16 did not.  The bound is stated as a 768-thread maximum (65536 / 768 -> 80 registers)
// because big mode launches the same instantiations with one 512-thread CTA per SM.
constexpr int EXTEND_SMEM_MAX_THREADS = 768;
// PRIMARY: camera rays (origin anywhere) -> exact slab arithmetic; later bounces start on scene surfaces -> FMA slabs.
// UNIFORM: one material class and no pre-pass (sc.uniform_class, UniformTally); otherwise ClassTally and k_volume_decide's verdicts.
template <bool SMEM, bool PRIMARY, bool UNIFORM>
__global__ void __launch_bounds__(SMEM ? EXTEND_SMEM_MAX_THREADS : 512) k_extend(DevScene sc, PathState ps, float4 *__restrict__ hit_out, uint32_t *__restrict__ ctrl,
                                                                                  uint32_t parity, Queues q, int max_stack, WaveCounters *ctr) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    const int stride = blockDim.x;
    BvhView bv;
    if (SMEM) bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar);
    else bv = global_bvh(sc);
    const uint32_t n = ctrl[parity];
    if (blockIdx.x == 0 && threadIdx.x == 0) ctrl_reset_parity(ctrl, parity ^ 1u);   // counters of the NEXT bounce (last used two bounces ago)
    uint32_t *qc = ctrl + CTRL_Q + 8u * parity;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t K = min(8u, max(1u, n / (gridDim.x * blockDim.x * 2u)));
    const uint32_t seg_paths = K * blockDim.x, n_seg = (n + seg_paths - 1u) / seg_paths;
    for (uint32_t seg = blockIdx.x; seg < n_seg; seg += gridDim.x) {
        const uint32_t base_i = seg * seg_paths + (threadIdx.x & ~31u);     // first path of this warp in iteration 0
        UniformTally ut; ClassTally ct;
        uint32_t i = base_i + lane;
        float4 o4 = make_float4(0, 0, 0, 0), d4 = o4;
        if (i < n) { o4 = ps.org_pdf[i]; d4 = ps.dir_rng[i]; }
        for (uint32_t it = 0; it < K; it++, i += blockDim.x) {
            if (base_i + it * blockDim.x >= n) { if (!UNIFORM) ct.skip(it); continue; }   // warp-uniform
            const bool active = i < n;
            bool hit = false;
            uint32_t code = Q_NONE;
            float4 o4n = make_float4(0, 0, 0, 0), d4n = o4n;
            if (it + 1u < K && i + blockDim.x < n) { o4n = ps.org_pdf[i + blockDim.x]; d4n = ps.dir_rng[i + blockDim.x]; }   // software pipelining of the state loads
            const uint32_t pre = (!UNIFORM && active && sc.pre_pass) ? __float_as_uint(hit_out[i].w) : 0u;   // k_volume_decide's verdict on this segment
            if (!UNIFORM && pre == VOLUME_EVENT) {
                code = 1u + MC_GENERAL;                                     // scattered inside a volume / the atmosphere: no TraceRay, SH/RayGen.slang:86-90
            } else if (!UNIFORM && pre == DEAD_EVENT) {
                code = Q_NONE;                                              // finished in k_volume_decide (below the planet surface): nothing to queue
            } else if (active) {
                const float3 rd = normalize_ray(f3(d4));                    // SH/RayGen.slang:70
                HitRec h;
                hit = bvh_trace<SMEM, false, false, false, !PRIMARY>(bv, f3(o4), rd, 0.01f, 100000.0f, h, stack, stride, max_stack);   // :71-72
                hit_out[i] = make_float4(h.t, h.u, h.v, __uint_as_float(h.gid));
                if (!UNIFORM) code = hit ? hit_code(sc, h.gid) : 0u;
            }
            o4 = o4n; d4 = d4n;
            if (UNIFORM) ut.add(it, lane, active, hit); else ct.add(it, lane, code);
        }
        if (UNIFORM) ut.flush(K, base_i, blockDim.x, lane, qc, sc.uniform_class, q); else ct.flush(K, base_i, blockDim.x, lane, qc, q);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&ctr->extend_rays, (unsigned long long)n);
}

// ------------------------------------------------------------------------------------------------
// k_camera : k_raygen and the camera rays' k_extend in one kernel, for scenes whose BVH is staged in shared memory and walked one ray per
//            thread, without a pre-pass (no volumes, no atmosphere).  Each path's state is written for the shading kernels as k_raygen writes
//            it, but the ray is traced from registers instead of being read back: the closest-hit query of k_extend<true, true, .>
//            (normalize_ray, exact slabs, tmin 0.01, tmax 1e5).  The hit record goes to hit_out, the path to the queues of parity 0.
//            The control block is cleared on the stream before the launch (launch_camera): the appends of other CTAs may run before
//            block 0 does.  With WAVE_IMPLIED and WAVE_STORE (the default pipeline) a path costs 36 B of stores: dir_rng, the hit record,
//            the queue entry.
// ------------------------------------------------------------------------------------------------
// 64 registers: 4 CTAs of 256 threads per SM (big mode: 2 of 512).  ADAPTIVE: as k_raygen<true> (P = active count, `active_px` unused otherwise).
template <bool UNIFORM, bool ADAPTIVE>
__global__ void __launch_bounds__(512, 2) k_camera(DevScene sc, DevConfig cfg, const DevDispatch *__restrict__ disp, uint32_t n_disp, uint32_t P,
                                                   uint32_t first_sample, uint32_t flags, const uint32_t *__restrict__ rng_carry, PathState ps,
                                                   float4 *__restrict__ sample_buf, float4 *__restrict__ hit_out, uint32_t *__restrict__ ctrl,
                                                   Queues q, int max_stack, WaveCounters *ctr, const uint32_t *__restrict__ active_px) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    const int stride = blockDim.x;
    const BvhView bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar);
    // Flat scenes: the origin-only part of every triangle test, for rays from the camera position (flat_fixed_trace).  A warp uses the table
    // only when all its rays start bit for bit there (always without depth of field); otherwise it walks the scene like k_extend.
    __shared__ float4 fixed_tab[4 * FLAT_FIXED_MAX];
    __shared__ float4 fixed_eye;
    const bool fixed = bv.n_flat != 0u && bv.n_flat <= FLAT_FIXED_MAX;
    if (fixed) {
        const float3 eye = camera_eye(cfg);
        for (uint32_t s = threadIdx.x; s < bv.n_flat; s += blockDim.x) flat_fixed_entry(bv, s, eye, fixed_tab);
        if (threadIdx.x == 0) fixed_eye = make_float4(eye.x, eye.y, eye.z, 0.0f);
        __syncthreads();
    }
    const uint32_t n = n_disp * P;
    if (blockIdx.x == 0 && threadIdx.x == 0) {                              // nothing in this launch reads ctrl[0]: the first k_shade_* kernels do
        ctrl[0] = n;
        atomicAdd(&ctr->paths, (unsigned long long)n); atomicAdd(&ctr->extend_rays, (unsigned long long)n);
    }
    uint32_t *qc = ctrl + CTRL_Q;                                           // queues of parity 0
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t K = min(8u, max(1u, n / (gridDim.x * blockDim.x * 2u)));
    // the segments of k_extend, walked by the warp's first path (one loop register fewer: 64 registers without spilling)
    const uint32_t seg_paths = K * blockDim.x;
    for (uint32_t base_i = blockIdx.x * seg_paths + (threadIdx.x & ~31u); base_i < n; base_i += gridDim.x * seg_paths) {
        UniformTally ut; ClassTally ct;
        uint32_t i = base_i + lane;
        for (uint32_t it = 0; it < K; it++, i += blockDim.x) {
            if (base_i + it * blockDim.x >= n) { if (!UNIFORM) ct.skip(it); continue; }   // warp-uniform
            const bool active = i < n;
            bool hit = false;
            uint32_t code = Q_NONE;
            float3 o = f3(0.0f), d = o;
            if (active) camera_path<ADAPTIVE>(cfg, disp, P, first_sample, flags, rng_carry, ps, sample_buf, i, o, d, active_px);
            bool at_eye = false;
            if (fixed) {
                const float4 e = fixed_eye;
                at_eye = __all_sync(0xFFFFFFFFu, !active || (__float_as_uint(o.x) == __float_as_uint(e.x) && __float_as_uint(o.y) == __float_as_uint(e.y) &&
                                                              __float_as_uint(o.z) == __float_as_uint(e.z)));
            }
            if (active) {                                                   // overhang pixels of a chunked dispatch are born dead and still traced, as in k_extend
                const float3 rd = normalize_ray(d);                         // SH/RayGen.slang:70-72
                HitRec h;
                hit = at_eye ? flat_fixed_trace(fixed_tab, bv.n_flat, rd, 0.01f, 100000.0f, h)
                             : bvh_trace<true, false, false, false, false>(bv, o, rd, 0.01f, 100000.0f, h, stack, stride, max_stack);
                hit_out[i] = make_float4(h.t, h.u, h.v, __uint_as_float(h.gid));
                if (!UNIFORM) code = hit ? hit_code(sc, h.gid) : 0u;
            }
            if (UNIFORM) ut.add(it, lane, active, hit); else ct.add(it, lane, code);
        }
        if (UNIFORM) ut.flush(K, base_i, blockDim.x, lane, qc, sc.uniform_class, q); else ct.flush(K, base_i, blockDim.x, lane, qc, q);
    }
}

// SH/RayGen.slang:116-128: an unsplit path adds all of pathLight, a path split by an atmosphere event only its colour channel
__device__ __forceinline__ void add_path_light(float4 &acc, float3 rad, int channel) {
    if (channel < 0) { acc.x += rad.x; acc.y += rad.y; acc.z += rad.z; }
    else if (channel == 0) acc.x += rad.x; else if (channel == 1) acc.y += rad.y; else acc.z += rad.z;
}
// A finished path (SH/RayGen.slang:116-128): its radiance is folded into its sample slot, its RNG state carried to the next sub-wave.
// WAVE_STORE: the slot holds nothing yet (a cleared slot holds zeros), so the sum starts from zeros instead of a load -- the same bits.
// Without WAVE_CARRY no later sub-wave reads rng_carry.
__device__ __forceinline__ void finish_path_slot(uint32_t flags, uint32_t slot, float3 rad, int channel, uint32_t rng_state,
                                                 float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry) {
    const bool ok = !isinf(rad.x) && !isinf(rad.y) && !isinf(rad.z) && !isnan(rad.x) && !isnan(rad.y) && !isnan(rad.z);   // :116
    float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (!(flags & WAVE_STORE)) acc = sample_buf[slot];
    if (ok) add_path_light(acc, rad, channel);
    sample_buf[slot] = acc;
    if (flags & WAVE_CARRY) rng_carry[slot] = rng_state;
}
// SH/Miss.slang:8-76 + the ray-gen epilogue for a path whose segment missed (k_shade_miss)
__device__ __forceinline__ void finish_missed_path(const DevScene &sc, const DevConfig &cfg, float3 dir, uint32_t rng_state, float4 t4, float4 r4, float payPDF,
                                                   uint32_t flags, float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry) {
    const uint32_t depth = __float_as_uint(t4.w) & DEPTH_MASK;
    const int channel = dflags_channel(__float_as_uint(t4.w));
    const float3 em = f3(miss_emission(sc, cfg, dir, depth, payPDF));
    // SH/RayGen.slang:92-102 with payload.Depth == MAX_DEPTH (!= 1): the contribution is always luminance-clamped (Q3)
    float3 contribution = em * f3(t4);
    const float lum = dot(contribution, f3(0.212671f, 0.715160f, 0.072169f));
    contribution = contribution * (cfg.MaxLuminance / fmaxf(lum, cfg.MaxLuminance));
    const float3 rad = f3(r4) + contribution;
    Rng rng; rng.s = rng_state;
    (void)rng.next();                                                       // the Russian-roulette draw of this segment (:111) still advances the stream
    finish_path_slot(flags, __float_as_uint(r4.w), rad, channel, rng.s, sample_buf, rng_carry);
}

// ------------------------------------------------------------------------------------------------
// k_shade_miss : SH/Miss.slang:8-76 for the miss queue.  A miss always ends the path (Depth = MAX_DEPTH), so the
//                ray-gen epilogue (SH/RayGen.slang:92-128) is applied here and the path never reaches k_connect.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_shade_miss(DevScene sc, DevConfig cfg, PathState ps, uint32_t *__restrict__ ctrl, uint32_t parity,
                                                     const uint32_t *__restrict__ q_miss, float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry,
                                                     WaveCounters *ctr, uint32_t flags) {
    const uint32_t n = ctrl[CTRL_Q + 8u * parity];
    const bool implied = (flags & WAVE_IMPLIED) != 0u;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t i = q_miss[j];
        const float4 d4 = ps.dir_rng[i];
        float4 t4, r4; float pdf;
        if (implied) { t4 = camera_implied_thr_depth(true); r4 = camera_implied_rad_slot(i); pdf = CAMERA_IMPLIED_PDF; }
        else { t4 = ps.thr_depth[i]; r4 = ps.rad_slot[i]; pdf = ps.org_pdf[i].w; }
        finish_missed_path(sc, cfg, f3(d4), __float_as_uint(d4.w), t4, r4, pdf, flags, sample_buf, rng_carry);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { atomicAdd(&ctr->misses, (unsigned long long)n); atomicAdd(&ctr->shade_invocations, (unsigned long long)n); }
}

// SH/RayGen.slang:92-113 for a path that was shaded at a hit, in two parts: path_roulette (throughput update, Russian roulette (Q4), loop
// condition) does not depend on the NEE terms; path_radiance (contribution, luminance clamp unless Depth == 1 (Q3), radiance; a finished path is folded into its sample slot, :116-128)
// runs once they are joined.  k_connect calls both in sequence.
// The join and every product / sum of the epilogue are written with explicitly rounded operations, in the form k_connect compiled to when
// its inputs came from memory: a value that stays in registers (the fused kernels) must not be contracted into an FMA that the unfused
// pipeline, whose NEE terms and BxDF pass through HBM, cannot form.  Fused and unfused images are then bit-identical.
__device__ __forceinline__ float3 add_rn(float3 a, float3 b) { return f3(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z)); }
__device__ __forceinline__ float3 mul_rn(float3 a, float3 b) { return f3(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y), __fmul_rn(a.z, b.z)); }
__device__ __forceinline__ float3 nee_join(float3 emitted, float3 c) { return add_rn(emitted, c); }   // payload.Emitted += NEE term (sky, then light)
__device__ __forceinline__ bool path_roulette(const DevConfig &cfg, float4 b4, uint32_t newDepth, float4 thr4, Rng &rng, float3 &thr) {
    thr = mul_rn(f3(thr4), f3(b4) / b4.w);
    float p = fmaxf(thr.x, fmaxf(thr.y, thr.z));
    p = fminf(p, 1.0f);
    const float u = rng.next();                                             // Q4
    bool alive = !(p < u);
    if (alive) thr = thr / p;
    return alive && (newDepth < cfg.MaxDepth);                              // loop condition :66
}
__device__ __forceinline__ float3 path_radiance(const DevConfig &cfg, float3 emitted, uint32_t newDepth, int channel, float4 thr4, float4 r4, bool alive, uint32_t rng_state,
                                                uint32_t flags, float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry) {
    float3 contribution = mul_rn(emitted, f3(thr4));
    if (newDepth != 1u) {                                                   // Q3: dot(contribution, luminance weights)
        const float lum = __fmaf_rn(contribution.z, 0.072169f, __fmaf_rn(contribution.x, 0.212671f, __fmul_rn(contribution.y, 0.715160f)));
        const float scale = cfg.MaxLuminance / fmaxf(lum, cfg.MaxLuminance);
        contribution = mul_rn(contribution, f3(scale));
    }
    const float3 rad = add_rn(f3(r4), contribution);
    if (!alive) finish_path_slot(flags, __float_as_uint(r4.w), rad, channel, rng_state, sample_buf, rng_carry);   // path finished: :116-128
    return rad;
}

// ------------------------------------------------------------------------------------------------
// k_shade_hit<CLASS, VOL, FUSE> : SH/ClosestHit.slang:20-378 for the hit queue of one material class.
//   !FUSE  writes the new ray + payload in place and <= 2 NEE shadow requests; k_connect (or k_shadow_dyn + k_connect) finishes the bounce.
//   FUSE   for scenes whose BVH is staged in shared memory (no volumes): each NEE request is traced the moment it is built (one copy of
//          the any-hit traversal inside the rolled NEE loop), then SH/RayGen.slang:92-113 runs in the same thread and the survivor is
//          written compacted to the other PathState buffer -- no request / payload round trip through HBM, no k_connect.
// ------------------------------------------------------------------------------------------------
#ifndef SHADE_MIN_BLOCKS
#define SHADE_MIN_BLOCKS 5
#endif
// The fused form runs 128-thread CTAs (4 per SM) or, in big mode, one 512-thread CTA per SM (BVHs of 64 KiB and more, which fit shared memory
// only once per SM).  Both bounds cap it at 128 registers, without spills (a 5 x 128 bound's 96-register cap spills 84-140 B).
template <uint32_t CLASS, bool VOL, bool FUSE>   // VOL: the scene has AABB volumes (volumes.cuh) -- volume events in the hit queue are skipped, NEE terms get the transmittance
__global__ void __launch_bounds__(FUSE ? 512 : 128, FUSE ? 1 : SHADE_MIN_BLOCKS) k_shade_hit(DevScene sc, DevConfig cfg, PathState ps, PathState dst, ShadeOut so,
                                                    const float4 *__restrict__ hit_in,
                                                    uint32_t *__restrict__ ctrl, uint32_t parity, Queues q,
                                                    float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry, int max_stack, WaveCounters *ctr,
                                                    uint32_t flags) {
    constexpr uint32_t LOBES = class_lobes(CLASS);
    // bounce 0 behind k_camera: only dir_rng of the path state was written.  Fused forms only: inferring the state in the unfused form (held to
    // 96 registers, already spilling) costs it spill traffic, so the engine does not set WAVE_IMPLIED for the unfused pipeline.
    const bool implied = FUSE && (flags & WAVE_IMPLIED) != 0u;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    const int stride = blockDim.x;
    BvhView bv;
    if (FUSE) bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar);
    const uint32_t n = ctrl[CTRL_Q + 8u * parity + 1u + CLASS];
    const uint32_t *__restrict__ q_hit = q.hit + (size_t)CLASS * q.cap;
    uint32_t *n_next_ptr = ctrl + (parity ^ 1u);
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t n_med = 0, n_shadow = 0;
    const float4 zero4 = make_float4(0, 0, 0, 0);
    // The queue entry and the hit record of the NEXT path of this thread are fetched one iteration ahead (two dependent DRAM
    // round trips off the critical path for 5 registers); its path-state lines are pulled towards L2 meanwhile.
    const uint32_t jstep = gridDim.x * blockDim.x;
    uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t i_nx = 0; float4 h4_nx = zero4;
    if (j < n) { i_nx = q_hit[j]; h4_nx = hit_in[i_nx]; }
    const uint32_t n_loop = FUSE ? ((n + 31u) & ~31u) : n;                  // fused: warps stay converged for the compaction collectives
    for (; j < n_loop; j += jstep) {
        const bool valid = j < n;
        // ---- results of the shading part, consumed by the fused tail
        bool shaded = false;                                                // this lane holds a path whose bounce must be finished (fused)
        float3 emitted = f3(0.0f), newO = f3(0.0f), newD = f3(0.0f);
        float4 b4 = zero4; uint32_t newDflags = 0u; Rng rng; rng.s = 0u;
        bool entered = false;
        const DevMaterial *cmp = nullptr;
        const uint32_t i = i_nx;
        if (valid) do {
            const float4 h4 = h4_nx;
            // implied: the origin is never read at Depth 0 outside a medium (the medium branch and the emission MIS need Depth != 0)
            const float4 o4 = implied ? make_float4(0.0f, 0.0f, 0.0f, CAMERA_IMPLIED_PDF) : ps.org_pdf[i], d4 = ps.dir_rng[i];
            const uint32_t dflags = implied ? __float_as_uint(camera_implied_thr_depth(true).w) : __float_as_uint(ps.thr_depth[i].w);
            if (j + jstep < n) {
                i_nx = q_hit[j + jstep]; h4_nx = hit_in[i_nx];
                if (!implied) asm volatile("prefetch.global.L2 [%0];" ::"l"(ps.org_pdf + i_nx));
                asm volatile("prefetch.global.L2 [%0];" ::"l"(ps.dir_rng + i_nx));
                if (!implied) asm volatile("prefetch.global.L2 [%0];" ::"l"(ps.thr_depth + i_nx));
                if (FUSE && !implied) asm volatile("prefetch.global.L2 [%0];" ::"l"(ps.rad_slot + i_nx));   // read by the path epilogue
            }
            const uint32_t depth = dflags & DEPTH_MASK;
            const uint32_t chanBits = dflags & CHANNEL_MASK;           // colour channel of a path split by an atmosphere event (0 = unsplit)
            const bool inMedium = (dflags >> 31) != 0u;
            const float3 payOrigin = f3(o4), payDir = f3(d4);
            const float payPDF = o4.w;
            rng.s = __float_as_uint(d4.w);
            const uint32_t gid = __float_as_uint(h4.w);                        // global triangle id of the hit
            if (VOL && gid == VOLUME_EVENT) break;                          // a volume scattering event: k_shade_volume

            // The sky-NEE draws are the first draws of a hit outside a medium: take them now and put the alias-table load in flight.
            EnvPick ep;
            const bool envEarly = cfg.EnableSkyMIS && !inMedium && !cfg.EnableAtmosphere;   // (with the atmosphere the sky sample is the sun disk: no table load to hide)
            if (envEarly) sample_env_begin(sc, rng, ep);

            const float3 rd = normalize(payDir);                                // WorldRayDirection()
            float4 g[7];                                                        // one 112-B gather: vertices + ids of the hit triangle
            {
                const float4 *gp = reinterpret_cast<const float4 *>(sc.shade_tris + gid);
                #pragma unroll
                for (int qq = 0; qq < 7; qq++) g[qq] = __ldg(gp + qq);
            }
            const uint32_t inst = __float_as_uint(g[0].w);
            const DevInstance &in = sc.instances[inst];
            const DevMaterial &cm = sc.materials[__float_as_uint(g[2].w)];
            cmp = &cm;
            Surface sf;
            surface_init(sf, sc, cfg, in, g, h4.y, h4.z, rd, cm);
            Mat m;
            material_init(m, sc, cfg, cm, sf);
            const bool isLight = m.EmissiveColor.x > 0.0f || m.EmissiveColor.y > 0.0f || m.EmissiveColor.z > 0.0f;   // :65
            surface_rotate_tangents(sf, m.AnisotropyRotation);                  // :67

            bool newInMedium = inMedium;
            if (inMedium) {                                                     // :80-116 (Q6)
                const float4 med = ps.medium[i]; const float med_g = ps.medium_g[i];
                const float dist = length(payOrigin - sf.WorldPos);
                if (med_g == 1.0f) {
                    // Beer-law BxDF is overwritten below (:323) -- nothing observable happens here.
                } else {
                    const float sd = -logf(rng.next()) / med.w;
                    if (sd < dist) {
                        const float3 no = payOrigin + payDir * sd;
                        const float3 nd = sample_henyey_greenstein(rng, payDir, med_g);
                        n_med++;
                        if (FUSE) {                                             // Depth and InMedium unchanged, no NEE, stale PDF (Q6)
                            newO = no; newD = nd; b4 = make_float4(med.x, med.y, med.z, payPDF); newDflags = dflags; shaded = true;
                        } else {
                            ps.org_pdf[i] = make_float4(no.x, no.y, no.z, payPDF);
                            ps.dir_rng[i] = make_float4(nd.x, nd.y, nd.z, __uint_as_float(rng.s));
                            so.bxdf_pdf[i] = make_float4(med.x, med.y, med.z, payPDF);
                            so.e0[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(dflags));
                        }
                        break;
                    }
                }
            }

            // emission :265-317 (no RNG draws: evaluated before the NEE/BSDF loop so the corner positions and the ray origin die here)
            emitted = hit_emission(sc, cfg, in, sf, m, isLight, depth, payOrigin, payPDF);

            float3 V = normalize(-rd);
            V = sf.world_to_tangent(V);
            BsdfCtx bc;
            bsdf_ctx_init<LOBES>(bc, m, sc, cfg, V);
            // Three uses of EvaluateBSDF(V, .) per hit -- sky NEE (:125-147, :326-358), light NEE (:154-184, :360-372) and the sampled
            // direction (SampleBSDF :94-165) -- run as ONE rolled loop in the reference's RNG order (sky draws, light draws, BSDF draws):
            // a single copy of the BSDF code stays in the kernel, and each NEE request is built and stored (or, fused, traced) inside its
            // own iteration so its direction / radiance / pdf registers die there.
            Eval evS; evS.BxDF = f3(0.0f); evS.PDF = 0.0f;
            float3 Ls = f3(0.0f); bool validDir = false;
            uint32_t reqMask = 0u;                                              // bit 0: sky request stored, bit 1: light request stored
            #pragma unroll 1
            for (int k = 0; k < 3; k++) {
                float3 toW = f3(0.0f), dk = f3(0.0f); float4 lv = zero4; uint32_t lgid = 0xFFFFFFFFu;
                bool need = false;
                if (k == 0) {
                    if (cfg.EnableSkyMIS) {
                        if (cfg.EnableAtmosphere) sample_sun_disk(cfg, rng, toW, lv);   // ImportanceSampleSky under ENABLE_ATMOSPHERE (SH/Sampler.slang:465-476)
                        else {
                            if (!envEarly) sample_env_begin(sc, rng, ep);
                            sample_env_finish(sc, cfg, ep, toW, lv);
                        }
                        lv.x *= cfg.EnvironmentIntensity; lv.y *= cfg.EnvironmentIntensity; lv.z *= cfg.EnvironmentIntensity;   // Q7
                        dk = sf.world_to_tangent(toW);
                        need = lv.w > 0.0f;
                    }
                } else if (k == 1) {
                    if (cfg.EnableMeshMIS && !isLight) {
                        sample_emissive(sc, rng, sf.WorldPos, toW, lv, lgid);
                        if (lv.w > 0.0f) { dk = sf.world_to_tangent(toW); need = true; }
                    }
                } else {
                    const float3 H = ggx_sample_vndf(rng, V, m.Ax, m.Ay);           // :191-204
                    validDir = sample_bsdf_direction<LOBES>(m, bc, rng, V, H, Ls);
                    dk = Ls; need = validDir;
                }
                Eval e; e.BxDF = f3(0.0f); e.PDF = 0.0f;
                if (need) e = eval_bsdf<LOBES>(m, bc, cfg, V, dk);
                if (k == 2) { evS = e; break; }
                // NEE term (added iff the shadow query allows) :326-372.  With the atmosphere on, the sky query is issued even when its term is zero:
                // k_connect draws the transmittance walk whenever the sun is VISIBLE (SH/ClosestHit.slang:335-349 sits outside the pdf tests)
                const bool contributes = need && e.PDF > 0.0f;
                if (contributes || (k == 0 && (cfg.EnableAtmosphere || (VOL && sc.n_grids)) && cfg.EnableSkyMIS)) {   // grid volumes: same reason (:332-333)
                    const float3 c = contributes ? nee_term(e, lv) : f3(0.0f);
                    // :139, :171 -- rounded like the unfused kernel, which stores the origin (product and sum apart, whatever the kernel around it)
                    const float3 ro = add_rn(sf.WorldPos, (k == 0) ? mul_rn(sf.Normal, f3(1e-5f)) : mul_rn(toW, f3(1e-2f)));
                    if (FUSE) {
                        //   sky   (SH/ClosestHit.slang:139 + :326-358): any hit in (1e-4, 1e6) occludes;
                        //   light (:171-176 + :360-372): the closest hit must be the sampled triangle.  Equivalent occlusion form: the ray hits
                        //         that triangle at tL and nothing lies in front of it (ties at tL resolve to the lower triangle id, exactly like
                        //         the closest-hit query) -- bounded by tL and free to stop at the first occluder.
                        // Both run through the TARGET any-hit query: for the sky ray target = 0xFFFFFFFF and tmax_test = tmax = 1e6.
                        float tmax = 1000000.0f, tmax_test = 1000000.0f; bool go = true;
                        if (k == 1) {
                            const float4 *tp = bv.tris + (size_t)__ldg(sc.tri_slot + lgid) * 3;
                            const float4 ta = tp[0], tb = tp[1], tc = tp[2];
                            float tL, uL, vL;
                            go = tri_test(f3(ta), f3(tb), f3(tc), ro, toW, 0.0001f, 1000000.0f, tL, uL, vL);
                            tmax = tL; tmax_test = light_tmax_test(tL);
                        }
                        n_shadow++;
                        if (go) {
                            HitRec hs;
                            const bool occluded = bvh_trace<true, true, false, true, true>(bv, ro, toW, 0.0001f, tmax, hs, stack, stride, max_stack, nullptr, nullptr, lgid, tmax_test);
                            if (!occluded) emitted = nee_join(emitted, c);
                        }
                    } else {
                        float4 *const po = (k == 0) ? so.sky_o : so.lit_o, *const pd = (k == 0) ? so.sky_d : so.lit_d, *const pc = (k == 0) ? so.sky_c : so.lit_c;
                        po[i] = make_float4(ro.x, ro.y, ro.z, 1.0f);
                        pd[i] = make_float4(toW.x, toW.y, toW.z, __uint_as_float(lgid));        // .w of the light request: id of the sampled triangle
                        pc[i] = make_float4(c.x, c.y, c.z, 0.0f);
                        reqMask |= 1u << k;
                    }
                }
            }
            BSample ss;
            ss.L = validDir ? Ls : f3(0.0f); ss.BxDF = evS.BxDF; ss.PDF = evS.PDF;
            const bool wasRefracted = ss.L.z < 0.0f;
            const float3 scatterW = sf.tangent_to_world(ss.L);
            if (!wasRefracted && dot(scatterW, sf.GeometryNormal) < 0.0f) { ss.PDF = 0.0f; ss.BxDF = f3(0.0f); }   // :220-225
            if (wasRefracted && sf.HitFromInside) newInMedium = false;          // :227-238
            else if (wasRefracted && !sf.HitFromInside) {                       // entering: the medium parameters are re-read from the material
                newInMedium = true;                                             // record here instead of being carried through the loop above
                entered = true;
                if (!FUSE) {
                    const b200pt_material &mm = cm.m;
                    const float3 mc = cfg.FurnaceTestMode ? f3(1.0f) : f3(mm.MediumColor[0], mm.MediumColor[1], mm.MediumColor[2]);   // SH/Material.slang:78-86
                    ps.medium[i] = make_float4(mc.x, mc.y, mc.z, mm.MediumDensity); ps.medium_g[i] = mm.MediumAnisotropy;
                }
            }

            // payload write :319-324, :375-376
            const float off = -1e-3f * (wasRefracted ? 1.0f : 0.0f) + 1e-3f * (wasRefracted ? 0.0f : 1.0f);
            const float3 no = sf.WorldPos + sf.Normal * off;
            const bool invalid = ss.PDF <= 0.0f;
            const uint32_t newDepth = invalid ? PT_MAX_DEPTH + depth : depth + 1u;   // MAX_DEPTH*(invalid) + (Depth + 1*(!invalid))
            if (FUSE) {
                newO = no; newD = scatterW; b4 = make_float4(ss.BxDF.x, ss.BxDF.y, ss.BxDF.z, ss.PDF);
                newDflags = newDepth | chanBits | (newInMedium ? 0x80000000u : 0u); shaded = true;
            } else {
                if (VOL && reqMask && !sc.n_grids) {                            // volumes cast shadows on the NEE terms: transmittance from the NEW origin (:332-333, :364); with grid volumes k_connect walks it
                    if (reqMask & 1u) { const float T = volumes_transmittance(sc, no, f3(so.sky_d[i])); const float4 c = so.sky_c[i]; so.sky_c[i] = make_float4(c.x * T, c.y * T, c.z * T, 0.0f); }
                    if (reqMask & 2u) { const float T = volumes_transmittance(sc, no, f3(so.lit_d[i])); const float4 c = so.lit_c[i]; so.lit_c[i] = make_float4(c.x * T, c.y * T, c.z * T, 0.0f); }
                }
                ps.org_pdf[i] = make_float4(no.x, no.y, no.z, ss.PDF);
                ps.dir_rng[i] = make_float4(scatterW.x, scatterW.y, scatterW.z, __uint_as_float(rng.s));
                so.bxdf_pdf[i] = make_float4(ss.BxDF.x, ss.BxDF.y, ss.BxDF.z, ss.PDF);
                so.e0[i] = make_float4(emitted.x, emitted.y, emitted.z, __uint_as_float(newDepth | chanBits | (reqMask << 29) | (newInMedium ? 0x80000000u : 0u)));   // bits 29/30: stored shadow requests
            }
        } while (false);

        if (FUSE) {
            // ---- SH/RayGen.slang:92-113, then compaction into the other PathState buffer
            bool alive = false;
            float4 thr4 = zero4, r4 = zero4; float3 thr = f3(0.0f), rad = f3(0.0f);
            if (shaded) {
                if (implied) { thr4 = camera_implied_thr_depth(true); r4 = camera_implied_rad_slot(i); }
                else { thr4 = ps.thr_depth[i]; r4 = ps.rad_slot[i]; }
                alive = path_roulette(cfg, b4, newDflags & DEPTH_MASK, thr4, rng, thr);
            }
            if (shaded) rad = path_radiance(cfg, emitted, newDflags & DEPTH_MASK, dflags_channel(newDflags), thr4, r4, alive, rng.s, flags, sample_buf, rng_carry);
            const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, alive);
            if (ballot) {
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd(n_next_ptr, (uint32_t)__popc(ballot));
                base = __shfl_sync(0xFFFFFFFFu, base, 0);
                const uint32_t k = base + (uint32_t)__popc(ballot & ((1u << lane) - 1u));
                if (alive) {
                    dst.org_pdf[k] = make_float4(newO.x, newO.y, newO.z, b4.w);
                    dst.dir_rng[k] = make_float4(newD.x, newD.y, newD.z, __uint_as_float(rng.s));
                    dst.thr_depth[k] = make_float4(thr.x, thr.y, thr.z, __uint_as_float(newDflags));
                    dst.rad_slot[k] = make_float4(rad.x, rad.y, rad.z, r4.w);
                    if (newDflags >> 31) {
                        float4 mv; float mg;
                        if (entered) {
                            const b200pt_material &mm = cmp->m;
                            const float3 mc = cfg.FurnaceTestMode ? f3(1.0f) : f3(mm.MediumColor[0], mm.MediumColor[1], mm.MediumColor[2]);   // SH/Material.slang:78-86
                            mv = make_float4(mc.x, mc.y, mc.z, mm.MediumDensity); mg = mm.MediumAnisotropy;
                        } else { mv = ps.medium[i]; mg = ps.medium_g[i]; }
                        dst.medium[k] = mv; dst.medium_g[k] = mg;
                    }
                }
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) { n_med += __shfl_down_sync(0xFFFFFFFFu, n_med, o); n_shadow += __shfl_down_sync(0xFFFFFFFFu, n_shadow, o); }
    if (lane == 0 && n_med) atomicAdd(&ctr->medium_events, (unsigned long long)n_med);
    if (FUSE && lane == 0 && n_shadow) atomicAdd(&ctr->shadow_rays, (unsigned long long)n_shadow);
    if (blockIdx.x == 0 && threadIdx.x == 0) { atomicAdd(&ctr->shade_invocations, (unsigned long long)n); atomicAdd(&ctr->surface_hits, (unsigned long long)n); }
}

// ------------------------------------------------------------------------------------------------
// k_connect : shadow queries + SH/RayGen.slang:92-113 + stream compaction of the survivors (unfused pipeline; walks every hit queue)
// ------------------------------------------------------------------------------------------------
// WALKS: the atmosphere is on or the scene has grid volumes -- NEE terms then carry random transmittance walks (atmosphere.cuh, volumes.cuh); compiled out of
// the plain instantiations, whose register budget (64) they would double
template <bool SMEM, bool TRACE, bool WALKS = false>   // TRACE = false: k_shadow_dyn already cleared the request bits of occluded rays; only the join / roulette / compaction runs here
__global__ void __launch_bounds__(512) k_connect(DevScene sc, DevConfig cfg, PathState src, PathState dst, ShadeOut so,
                                                  uint32_t *__restrict__ ctrl, uint32_t parity, Queues q,
                                                  float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry,
                                                  int max_stack, WaveCounters *ctr, uint32_t flags) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    const int stride = blockDim.x;
    BvhView bv;
    if (SMEM && TRACE) bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar);
    else bv = global_bvh(sc);
    const HitSpan span = hit_span(ctrl, parity);
    const uint32_t n = span.n;                                              // paths that hit a surface this bounce (misses ended in k_shade_miss)
    uint32_t *n_next_ptr = ctrl + (parity ^ 1u);
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t n_shadow = 0;
    const uint32_t n_round = (n + 31u) & ~31u;                              // keep warps converged for the ballots
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_round; j += gridDim.x * blockDim.x) {
        const bool active = j < n;
        bool alive = false;
        float4 o4, d4, r4; uint32_t newDflags = 0; Rng rng; rng.s = 0;
        float3 thr = f3(0.0f), rad = f3(0.0f);
        uint32_t i = 0;
        if (active) {
            i = hit_entry(q, span, j);
            const float4 e4 = so.e0[i];
            uint32_t pending = (__float_as_uint(e4.w) >> 29) & 3u;         // bit 0: sky request, bit 1: light request (k_shade_hit)
            newDflags = __float_as_uint(e4.w) & 0x9FFFFFFFu;
            const uint32_t newDepth = newDflags & DEPTH_MASK;
            const int channel = dflags_channel(newDflags);
            float3 emitted = f3(e4);
            // Atmosphere: a visible sun costs the path a transmittance walk on its own RNG stream, BEFORE the roulette draw (SH/ClosestHit.slang:335-349,
            // SH/RayGen.slang:328-342,415-422) -- so the new origin and the RNG state are fetched up front instead of after the queries.
            // Grid volumes: the same for their ratio-tracking walks (SH/Volume.slang:448-517), sky then light; rayDepth is 0 after a surface hit (:333,:364),
            // VolumeDepth / VolumeDepth + 1 after a volume event (SH/RayGen.slang:326,361; k_shade_volume has already counted the event), VolumeDepth after
            // an atmosphere event, where the atmosphere walk comes FIRST (:415-421).
            const bool atm = WALKS && cfg.EnableAtmosphere != 0u, het = WALKS && sc.n_grids != 0u, walks = atm || het;
            float skyDepth = 0.0f, litDepth = 0.0f; bool atmEvent = false;
            if (walks) { o4 = src.org_pdf[i]; d4 = src.dir_rng[i]; rng.s = __float_as_uint(d4.w); }
            if (het && pending) {
                const float4 h4 = so.hit[i];
                if (__float_as_uint(h4.w) == VOLUME_EVENT) {
                    const float vd = (float)src.vol_depth[i];
                    if (__float_as_int(h4.y) >= 0) { skyDepth = vd - 1.0f; litDepth = vd; } else { skyDepth = vd; atmEvent = true; }
                }
            }
            auto sky_term = [&](float3 c, float3 dir) {
                if (atmEvent) { c = c * atm_transmittance_nee(cfg, rng, f3(o4), dir, channel); return c * volumes_transmittance_walk(sc, rng, f3(o4), dir, skyDepth); }
                if (het) c = c * volumes_transmittance_walk(sc, rng, f3(o4), dir, skyDepth);
                if (atm) c = c * atm_transmittance_nee(cfg, rng, f3(o4), dir, channel);
                return c;
            };
            // Request words are read when needed: the light request after the sky query, a contribution only if its ray came out
            // unoccluded, the path state after both queries -- little is live across the traversal loops.
            // (One resumable loop serving both rays of a lane, if-if style, was measured 1.6x SLOWER than two tight while-while loops.)
            //   sky   (SH/ClosestHit.slang:139 + :326-358): any hit in (1e-4, 1e6) occludes;
            //   light (:171-176 + :360-372): the closest hit must be the sampled triangle.  Equivalent occlusion form: the ray hits
            //         that triangle at tL and nothing lies in front of it (ties at tL resolve to the lower triangle id, exactly like
            //         the closest-hit query) -- bounded by tL and free to stop at the first occluder.
            if (TRACE) n_shadow += (pending & 1u) + (pending >> 1);
            if (!TRACE) {                                                   // surviving bits = unoccluded requests, joined in the reference's order
                if (pending & 1u) emitted = WALKS ? emitted + (walks ? sky_term(f3(so.sky_c[i]), f3(so.sky_d[i])) : f3(so.sky_c[i])) : nee_join(emitted, f3(so.sky_c[i]));
                if (pending & 2u) {
                    float3 c = f3(so.lit_c[i]);
                    if (het) c = c * volumes_transmittance_walk(sc, rng, f3(o4), f3(so.lit_d[i]), litDepth);
                    emitted = WALKS ? emitted + c : nee_join(emitted, c);
                }
                pending = 0u;
            }
            float4 so4 = make_float4(0, 0, 0, 0), sd4 = so4;
            if (pending & 1u) { so4 = so.sky_o[i]; sd4 = so.sky_d[i]; }
            if (pending & 1u) {
                HitRec h;
                const bool occluded = bvh_trace<SMEM, true, false, false, true>(bv, f3(so4), f3(sd4), 0.0001f, 1000000.0f, h, stack, stride, max_stack);
                if (!occluded) emitted = WALKS ? emitted + (walks ? sky_term(f3(so.sky_c[i]), f3(sd4)) : f3(so.sky_c[i])) : nee_join(emitted, f3(so.sky_c[i]));
            }
            if (pending & 2u) {
                const float4 lo4 = so.lit_o[i], ld4_ = so.lit_d[i];
                const uint32_t lgid = __float_as_uint(ld4_.w);
                const float4 *tp = bv.tris + (size_t)__ldg(sc.tri_slot + lgid) * 3;
                const float4 ta = ld4<SMEM>(tp), tb = ld4<SMEM>(tp + 1), tc = ld4<SMEM>(tp + 2);
                float tL, uL, vL;
                if (tri_test(f3(ta), f3(tb), f3(tc), f3(lo4), f3(ld4_), 0.0001f, 1000000.0f, tL, uL, vL)) {
                    HitRec h;
                    const bool occluded = bvh_trace<SMEM, true, false, true, true>(bv, f3(lo4), f3(ld4_), 0.0001f, tL, h, stack, stride, max_stack, nullptr, nullptr, lgid);
                    if (!occluded) {
                        float3 c = f3(so.lit_c[i]);
                        if (het) c = c * volumes_transmittance_walk(sc, rng, f3(o4), f3(ld4_), litDepth);
                        emitted = WALKS ? emitted + c : nee_join(emitted, c);   // (the walks' products may contract into the join: WALKS keeps its form)
                    }
                }
            }
            // the path state is fetched only now: nothing but the emission and the request bits is live across the traversal loop
            const float4 thr4 = src.thr_depth[i]; r4 = src.rad_slot[i];
            if (!walks) { o4 = src.org_pdf[i]; d4 = src.dir_rng[i]; rng.s = __float_as_uint(d4.w); }
            const float4 b4 = so.bxdf_pdf[i];
            alive = path_roulette(cfg, b4, newDepth, thr4, rng, thr);
            rad = path_radiance(cfg, emitted, newDepth, channel, thr4, r4, alive, rng.s, flags, sample_buf, rng_carry);
        }
        // ---- warp ballot + prefix-sum compaction of the live paths
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, alive);
        if (ballot) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(n_next_ptr, (uint32_t)__popc(ballot));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            if (alive) {
                const uint32_t k = base + (uint32_t)__popc(ballot & ((1u << lane) - 1u));
                dst.org_pdf[k] = o4;
                dst.dir_rng[k] = make_float4(d4.x, d4.y, d4.z, __uint_as_float(rng.s));
                dst.thr_depth[k] = make_float4(thr.x, thr.y, thr.z, __uint_as_float(newDflags));
                dst.rad_slot[k] = make_float4(rad.x, rad.y, rad.z, r4.w);
                if (newDflags >> 31) { dst.medium[k] = src.medium[i]; dst.medium_g[k] = src.medium_g[i]; }
                if (src.vol_depth) dst.vol_depth[k] = src.vol_depth[i];
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) n_shadow += __shfl_down_sync(0xFFFFFFFFu, n_shadow, o);
    if (lane == 0 && n_shadow) atomicAdd(&ctr->shadow_rays, (unsigned long long)n_shadow);
}

// ------------------------------------------------------------------------------------------------
// k_extend_dyn / k_shadow_dyn : the traversal kernels for scenes whose BVH does not fit in shared memory (bvh_dynfetch.cuh).
//   control block additions: ctrl[8+p] = fetch counter of k_extend_dyn, ctrl[10+p] = fetch counter of k_shadow_dyn (p = bounce parity)
// ------------------------------------------------------------------------------------------------
template <bool SMEM, bool PRIMARY, bool WIDE>   // WIDE: BVH4 nodes (sc.nodes4) instead of the BVH2
__global__ void __launch_bounds__(256) k_extend_dyn(DevScene sc, PathState ps, float4 *__restrict__ hit_out, uint32_t *__restrict__ ctrl, uint32_t parity,
                                                     Queues q, int max_stack, int thresh, WaveCounters *ctr) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    stack[0] = DYN_DONE;
    BvhView bv;
    if (SMEM) bv = stage_bvh_smem(sc, smem + (size_t)(max_stack + 1) * blockDim.x * sizeof(int), &bar);
    else bv = global_bvh(sc);
    const uint32_t n = ctrl[parity];
    if (blockIdx.x == 0 && threadIdx.x == 0) {                              // counters of the NEXT bounce (last used two bounces ago)
        ctrl_reset_parity(ctrl, parity ^ 1u);
        atomicAdd(&ctr->extend_rays, (unsigned long long)n);
    }
    uint32_t *qc = ctrl + CTRL_Q + 8u * parity;
    uint32_t *fetch = ctrl + 8u + parity;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t s_base = smem_u32(stack), s_step = blockDim.x * 4u, s_limit = s_base + (uint32_t)(max_stack + 1) * s_step;
    DynPool pool; pool.init(n, gridDim.x * (blockDim.x >> 5));
    DynRay r; r.cur = DYN_DONE; r.gid = DYN_NONE; r.t = 0.0f; r.u = 0.0f; r.v = 0.0f; r.s_top = s_base; r.n_spill = 0;
    int spill[WIDE ? DYN_SPILL : 1];
    const float4 *nodes4 = reinterpret_cast<const float4 *>(sc.nodes4);
    if (WIDE) bv.root = 0;                                                  // the BVH4 root is node 0 (bvh4_collapse_host)
    uint32_t i = DYN_NONE;
    while (true) {
        // ---- commit finished rays: hit record + miss / class queue entry (one multi-address atomic per refill event)
        const bool fin = (r.cur == DYN_DONE);
        const bool have = fin && i != DYN_NONE;
        const bool hit = have && r.gid != DYN_NONE;
        if (have && r.gid != VOLUME_EVENT) hit_out[i] = make_float4(hit ? r.t : -1.0f, r.u, r.v, __uint_as_float(r.gid));
        const uint32_t code = hit ? hit_code(sc, r.gid) : (have ? 0u : Q_NONE);
        if (__ballot_sync(0xFFFFFFFFu, have)) queue_append(code, i, qc, q, lane);
        // ---- refill
        const uint32_t need = __ballot_sync(0xFFFFFFFFu, fin);
        if (need) {
            const uint32_t idx = pool.take(need, lane, fetch);
            if (fin) {
                i = idx;
                const uint32_t pre = (i != DYN_NONE && sc.pre_pass) ? __float_as_uint(hit_out[i].w) : 0u;
                if (pre == VOLUME_EVENT) {
                    r.gid = VOLUME_EVENT;                                   // scattered inside a volume / the atmosphere (k_volume_decide): queued as a hit at the next commit, record kept
                } else if (pre == DEAD_EVENT) {
                    i = DYN_NONE;                                           // finished in k_volume_decide: the lane takes no ray this round
                } else if (i != DYN_NONE) {
                    const float4 o4 = ps.org_pdf[i], d4 = ps.dir_rng[i];
                    const float3 rd = normalize_ray(f3(d4));                // SH/RayGen.slang:70
                    dyn_init(r, f3(o4), rd, 0.01f, 100000.0f, 100000.0f, DYN_NONE, bv.root, s_base, s_step);   // :71-72
                }
            }
        }
        uint32_t act = __ballot_sync(0xFFFFFFFFu, r.cur != DYN_DONE);
        if (act == 0u) {                                                    // nobody traverses: drained, unless lanes hold volume events to commit
            if (__ballot_sync(0xFFFFFFFFu, i != DYN_NONE) == 0u) break;
            continue;
        }
        const int thr_now = pool.empty() ? 1 : thresh;
        do {
            act = dyn_round<SMEM, false, WIDE, !PRIMARY>(bv, nodes4, r, s_step, s_limit, spill, [] {});
        } while (__popc(act) >= thr_now);
    }
}

// Shadow requests of the hit queues, compacted per warp: ring entry = (path index << 1) | kind (0 sky, 1 light).
// An occluded ray clears its request bit in e0.w (bit 29 sky, bit 30 light); k_connect<.., false> joins the surviving requests.
constexpr size_t DYN_RING_BYTES = 8 * 128 * sizeof(uint32_t);              // per-CTA request rings of k_shadow_dyn (dynamic shared memory, after the stacks)
template <bool SMEM, bool WIDE>
__global__ void __launch_bounds__(256, 4) k_shadow_dyn(DevScene sc, ShadeOut so, uint32_t *__restrict__ ctrl, uint32_t parity,
                                                     Queues q, int max_stack, int thresh, WaveCounters *ctr) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    stack[0] = DYN_DONE;
    const size_t stack_bytes = (size_t)(max_stack + 1) * blockDim.x * sizeof(int);
    uint32_t *ring_all = reinterpret_cast<uint32_t *>(smem + stack_bytes);  // 128 entries per warp
    BvhView bv;
    if (SMEM) bv = stage_bvh_smem(sc, smem + stack_bytes + DYN_RING_BYTES, &bar);
    else bv = global_bvh(sc);
    const HitSpan span = hit_span(ctrl, parity);
    const uint32_t n = span.n;                                              // total hit-queue length of this bounce
    uint32_t *fetch = ctrl + 10u + parity;
    const uint32_t lane = threadIdx.x & 31u, lt = (1u << lane) - 1u;
    uint32_t *ring = ring_all + (threadIdx.x >> 5) * 128u;
    const uint32_t s_base = smem_u32(stack), s_step = blockDim.x * 4u, s_limit = s_base + (uint32_t)(max_stack + 1) * s_step;
    DynPool pool; pool.init(n, gridDim.x * (blockDim.x >> 5));
    DynRay r; r.cur = DYN_DONE; r.s_top = s_base; r.gid = DYN_NONE; r.t = 0.0f; r.n_spill = 0;
    int spill[WIDE ? DYN_SPILL : 1];
    const float4 *nodes4 = reinterpret_cast<const float4 *>(sc.nodes4);
    if (WIDE) bv.root = 0;
    uint32_t head = 0, tail = 0;                                            // warp-uniform ring cursors
    uint32_t n_shadow = 0;
    while (true) {
        const bool fin = (r.cur == DYN_DONE);
        const uint32_t need = __ballot_sync(0xFFFFFFFFu, fin);
        const uint32_t cnt = (uint32_t)__popc(need);
        // ---- top the ring up with the requests of the next 32 hit-queue entries until it covers the idle lanes
        while (tail - head < cnt && !pool.empty()) {
            const uint32_t j = pool.take(0xFFFFFFFFu, lane, fetch);
            uint32_t pend = 0, i = 0;
            if (j != DYN_NONE) { i = hit_entry(q, span, j); pend = (__float_as_uint(so.e0[i].w) >> 29) & 3u; }
            const uint32_t c = (pend & 1u) + (pend >> 1);
            uint32_t incl = c;
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o); if ((int)lane >= o) incl += y; }
            uint32_t w = tail + incl - c;
            if (pend & 1u) { ring[w & 127u] = i << 1; w++; }
            if (pend & 2u) ring[w & 127u] = (i << 1) | 1u;
            tail += __shfl_sync(0xFFFFFFFFu, incl, 31);
            n_shadow += c;
            __syncwarp();
        }
        // ---- hand requests to the idle lanes
        if (fin) {
            const uint32_t rank = (uint32_t)__popc(need & lt);
            if (rank < tail - head) {
                const uint32_t e = ring[(head + rank) & 127u];
                const uint32_t i = e >> 1;
                if (e & 1u) {                                               // light: SH/ClosestHit.slang:171-176 in its bounded any-hit form (k_connect)
                    const float4 lo4 = so.lit_o[i], ld4_ = so.lit_d[i];
                    const uint32_t lgid = __float_as_uint(ld4_.w);
                    const float4 *tp = bv.tris + (size_t)__ldg(sc.tri_slot + lgid) * 3;
                    const float4 ta = ld4<SMEM>(tp), tb = ld4<SMEM>(tp + 1), tc = ld4<SMEM>(tp + 2);
                    float tL, uL, vL;
                    if (tri_test(f3(ta), f3(tb), f3(tc), f3(lo4), f3(ld4_), 0.0001f, 1000000.0f, tL, uL, vL)) {
                        dyn_init(r, f3(lo4), f3(ld4_), 0.0001f, tL, light_tmax_test(tL), lgid, bv.root, s_base, s_step);
                        r.gid = e;
                    } else {
                        atomicAnd(reinterpret_cast<unsigned int *>(&so.e0[i].w), ~(1u << 30));
                    }
                } else {                                                    // sky: SH/ClosestHit.slang:139 -- any hit in (1e-4, 1e6) occludes
                    const float4 so4 = so.sky_o[i], sd4 = so.sky_d[i];
                    dyn_init(r, f3(so4), f3(sd4), 0.0001f, 1000000.0f, 1000000.0f, DYN_NONE, bv.root, s_base, s_step);
                    r.gid = e;
                }
            }
        }
        { const uint32_t avail = tail - head; head += cnt < avail ? cnt : avail; }
        __syncwarp();
        uint32_t act = __ballot_sync(0xFFFFFFFFu, r.cur != DYN_DONE);
        if (act == 0u) { if (tail == head && pool.empty()) break; else continue; }
        const int thr_now = (tail == head && pool.empty()) ? 1 : thresh;
        do {
            act = dyn_round<SMEM, true, WIDE, true>(bv, nodes4, r, s_step, s_limit, spill, [&] {   // occluded: drop the request
                atomicAnd(reinterpret_cast<unsigned int *>(&so.e0[r.gid >> 1].w), ~(1u << (29u + (r.gid & 1u))));
            });
        } while (__popc(act) >= thr_now);
    }
    for (int o = 16; o > 0; o >>= 1) n_shadow += __shfl_down_sync(0xFFFFFFFFu, n_shadow, o);
    if (lane == 0 && n_shadow) atomicAdd(&ctr->shadow_rays, (unsigned long long)n_shadow);
}

// ------------------------------------------------------------------------------------------------
// k_volume_decide / k_shade_volume : homogeneous AABB volumes (volumes.cuh; SH/RayGen.slang:162-380)
// ------------------------------------------------------------------------------------------------
template <bool SMEM>
__global__ void __launch_bounds__(256) k_volume_decide(DevScene sc, DevConfig cfg, PathState ps, ShadeOut so, const uint32_t *__restrict__ ctrl, uint32_t parity, int max_stack,
                                                        float4 *__restrict__ sample_buf, uint32_t *__restrict__ rng_carry) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    BvhView bv;
    if (SMEM) bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar);
    else bv = global_bvh(sc);
    const uint32_t n = ctrl[parity];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 o4 = ps.org_pdf[i], d4 = ps.dir_rng[i];
        const float3 o = f3(o4), d = f3(d4);
        Rng rng; rng.s = __float_as_uint(d4.w);
        if (cfg.EnableAtmosphere && atm_height(cfg, o) < 0.0f) {            // SH/RayGen.slang:76-84: below the surface of the planet -> the path loop breaks (no roulette draw)
            const float4 t4 = ps.thr_depth[i], r4 = ps.rad_slot[i];
            const float3 rad = f3(r4);
            const uint32_t slot = __float_as_uint(r4.w);
            const bool ok = !isinf(rad.x) && !isinf(rad.y) && !isinf(rad.z) && !isnan(rad.x) && !isnan(rad.y) && !isnan(rad.z);
            float4 acc = sample_buf[slot];
            if (ok) add_path_light(acc, rad, dflags_channel(__float_as_uint(t4.w)));
            sample_buf[slot] = acc; rng_carry[slot] = rng.s;
            so.hit[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(DEAD_EVENT));
            continue;
        }
        HitRec h;                                                           // GetDistanceToGeometry (SH/RTCommon.slang:86-100): payload.Direction as is, tmin 1e-5, tmax 1e6
        const bool found = bvh_trace<SMEM, false>(bv, o, d, 0.00001f, 1000000.0f, h, stack, (int)blockDim.x, max_stack);
        const float distanceToGeometry = found ? h.t : -1.0f;
        int vi = -1;
        const uint32_t dflags0 = __float_as_uint(ps.thr_depth[i].w);
        float sd = volumes_free_flight(sc, o, d, rng, (float)(dflags0 & DEPTH_MASK), vi);   // :164-209 (heterogeneous volumes: payload.Depth scales the density, :199)
        if (cfg.EnableAtmosphere) {                                         // :212-236: channel pick (while unsplit), delta tracking on that channel
            const uint32_t dflags = dflags0;
            int channel = dflags_channel(dflags);
            if (channel < 0) { const float pick = rng.next(); channel = pick < 0.33333f ? 0 : (pick < 0.66666f ? 1 : 2); }
            int component = -1;
            const float ta = atm_sample_scatter_distance(cfg, rng, o, d, channel, component);
            if (ta >= 0.0f && (ta < sd || sd < 0.0f)) {
                sd = ta; vi = -2 - component;                               // the atmosphere scattered first: event code -2 (Rayleigh) / -3 (Mie) / -4 (ozone)
                if (distanceToGeometry < 0.0f || sd < distanceToGeometry) {  // the event will happen: the ray is split to this channel from now on (:244)
                    float4 t4 = ps.thr_depth[i];
                    t4.w = __uint_as_float((dflags & ~CHANNEL_MASK) | ((uint32_t)(channel + 1) << CHANNEL_SHIFT));
                    ps.thr_depth[i] = t4;
                }
            }
        }
        ps.dir_rng[i] = make_float4(d4.x, d4.y, d4.z, __uint_as_float(rng.s));
        const bool ev = sd >= 0.0f && (distanceToGeometry < 0.0f || sd < distanceToGeometry);   // :236
        so.hit[i] = ev ? make_float4(sd, __int_as_float(vi), 0.0f, __uint_as_float(VOLUME_EVENT)) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
}

// EvaluateVolumeScatteringEvent (SH/RayGen.slang:265-380) / EvaluateAtmosphereScatteringEvent (:382-471) for the flagged entries of the hit queue
__global__ void __launch_bounds__(128) k_shade_volume(DevScene sc, DevConfig cfg, PathState ps, ShadeOut so, const uint32_t *__restrict__ ctrl, uint32_t parity,
                                                      Queues q, WaveCounters *ctr) {
    const uint32_t n = ctrl[CTRL_Q + 8u * parity + 1u + MC_GENERAL];          // volume events are queued with the general class (hit_code)
    const uint32_t *__restrict__ q_hit = q.hit + (size_t)MC_GENERAL * q.cap;
    uint32_t n_ev = 0;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t i = q_hit[j];
        const float4 h4 = so.hit[i];
        if (__float_as_uint(h4.w) != VOLUME_EVENT) continue;
        n_ev++;
        const float4 o4 = ps.org_pdf[i], d4 = ps.dir_rng[i];
        const uint32_t dflags = __float_as_uint(ps.thr_depth[i].w);
        Rng rng; rng.s = __float_as_uint(d4.w);
        const float3 dir = f3(d4);
        const float3 origin = f3(o4) + dir * h4.x;                          // :267 / :384
        const int code = __float_as_int(h4.y);
        if (code <= -2) {                                                   // ---- atmosphere event
            const int component = -2 - code;
            float3 newDir;
            if (component == 0) newDir = sample_rayleigh(rng, dir);
            else if (component == 1) newDir = sample_henyey_greenstein(rng, dir, 0.85f);
            else newDir = dir;                                              // ozone only absorbs
            const float C_MIE_ABS = 4.40f * 1e-6f, C_MIE = 3.996f * 1e-6f + 4.40f * 1e-6f;
            float3 bx; float pdf; uint32_t reqMask = 0u;
            if (cfg.EnableSkyMIS) {                                         // :403-446
                float3 toSun; float4 cp;
                sample_sun_disk(cfg, rng, toSun, cp);
                cp.x *= cfg.EnvironmentIntensity; cp.y *= cfg.EnvironmentIntensity; cp.z *= cfg.EnvironmentIntensity;
                const float3 col = f3(cp) / cp.w;
                float ph = 0.0f;
                if (component == 0) { ph = phase_rayleigh(dir, toSun); const float pn = phase_rayleigh(dir, newDir); bx = f3(pn); pdf = pn; }
                else if (component == 1) { ph = phase_hg(dir, toSun, 0.85f); const float att = C_MIE_ABS / C_MIE; const float pn = phase_hg(dir, newDir, 0.85f); bx = f3(pn * (1.0f - att)); pdf = pn; }
                else { bx = f3(0.0f); pdf = 1.0f; }
                // the sun query is always issued: its transmittance walk is drawn whenever the sun is visible (:415-422); k_connect multiplies by it
                const float Tv = volumes_transmittance_shade(sc, origin, toSun);
                const float3 c = (f3(Tv) * ph) * col;
                so.sky_o[i] = make_float4(origin.x, origin.y, origin.z, 1.0f);
                so.sky_d[i] = make_float4(toSun.x, toSun.y, toSun.z, __uint_as_float(0xFFFFFFFFu));
                so.sky_c[i] = make_float4(c.x, c.y, c.z, 0.0f);
                reqMask = 1u;
            } else {                                                        // :447-461
                if (component == 0) { const float pn = phase_rayleigh(dir, newDir); bx = f3(pn); pdf = pn; }
                else { const float att = C_MIE_ABS / C_MIE; bx = f3(phase_mie_approx(dir, newDir, 0.85f) * att); pdf = phase_hg(dir, newDir, 0.85f); }
            }
            const uint32_t newDepth = (dflags & DEPTH_MASK) + 1u;           // :470 (VolumeDepth untouched)
            ps.org_pdf[i] = make_float4(origin.x, origin.y, origin.z, pdf);
            ps.dir_rng[i] = make_float4(newDir.x, newDir.y, newDir.z, __uint_as_float(rng.s));
            so.bxdf_pdf[i] = make_float4(bx.x, bx.y, bx.z, pdf);
            so.e0[i] = make_float4(0.0f, 0.0f, 0.0f, __uint_as_float(newDepth | (dflags & (0x80000000u | CHANNEL_MASK)) | (reqMask << 29)));
            continue;
        }
        const DevVolume v = sc.volumes[code];
        const float3 color = f3(v.color_alpha);
        const int vdepth = (int)ps.vol_depth[i];
        const float3 emitted = f3(v.emis_droplet) + vol_temperature_emission(sc, v, rng, origin);   // :268
        float3 toSky = f3(0.0f), toLight = f3(0.0f); float4 sky = make_float4(0, 0, 0, 0), light = sky; uint32_t lgid = 0xFFFFFFFFu;
        if (cfg.EnableSkyMIS) {                                             // :273-287
            if (cfg.EnableAtmosphere) sample_sun_disk(cfg, rng, toSky, sky);
            else { EnvPick ep; sample_env_begin(sc, rng, ep); sample_env_finish(sc, cfg, ep, toSky, sky); }
            sky.x *= cfg.EnvironmentIntensity; sky.y *= cfg.EnvironmentIntensity; sky.z *= cfg.EnvironmentIntensity;   // Q7 again (:277)
        }
        if (cfg.EnableMeshMIS) sample_emissive(sc, rng, origin, toLight, light, lgid);   // :294-308
        const float3 newDir = vol_scatter_direction(sc.phase_function, v, rng, dir, vdepth);   // :311
        const float phaseS = vol_phase(sc.phase_function, v, dir, newDir, vdepth);             // :314
        uint32_t reqMask = 0u;
        // the two visibility queries of :280-306 become shadow requests; the phase-weighted, transmittance-attenuated MIS terms of
        // :319-369 are added by k_connect iff the query comes out clear (sky: any hit occludes; light: the sampled triangle must be the closest hit)
        if (cfg.EnableSkyMIS && sky.w > 0.0f) {
            const float ph = vol_phase(sc.phase_function, v, dir, toSky, vdepth);
            if (ph > 0.0f || cfg.EnableAtmosphere || sc.n_grids) {          // atmosphere / grid volumes: the query decides whether the transmittance walks are drawn (:326-342), even for a zero term
                const float T = volumes_transmittance_shade(sc, origin, toSky);
                const float3 c = ph > 0.0f ? ((f3(T) * (color * ph)) * (f3(sky) / sky.w)) * power_heuristic(sky.w, ph) : f3(0.0f);
                so.sky_o[i] = make_float4(origin.x, origin.y, origin.z, 1.0f);
                so.sky_d[i] = make_float4(toSky.x, toSky.y, toSky.z, __uint_as_float(0xFFFFFFFFu));
                so.sky_c[i] = make_float4(c.x, c.y, c.z, 0.0f);
                reqMask |= 1u;
            }
        }
        if (cfg.EnableMeshMIS && light.w > 0.0f) {
            const float ph = vol_phase(sc.phase_function, v, dir, toLight, vdepth);
            if (ph > 0.0f || sc.n_grids) {                                  // :361 sits outside the phase test
                const float T = volumes_transmittance_shade(sc, origin, toLight);
                const float3 c = ph > 0.0f ? ((f3(T) * (color * ph)) * (f3(light) / light.w)) * power_heuristic(light.w, ph) : f3(0.0f);
                so.lit_o[i] = make_float4(origin.x, origin.y, origin.z, 1.0f);
                so.lit_d[i] = make_float4(toLight.x, toLight.y, toLight.z, __uint_as_float(lgid));
                so.lit_c[i] = make_float4(c.x, c.y, c.z, 0.0f);
                reqMask |= 2u;
            }
        }
        const uint32_t newDepth = (dflags & DEPTH_MASK) + 1u;               // :377
        ps.org_pdf[i] = make_float4(origin.x, origin.y, origin.z, phaseS);  // payload.PDF = phase (:374)
        ps.dir_rng[i] = make_float4(newDir.x, newDir.y, newDir.z, __uint_as_float(rng.s));
        so.bxdf_pdf[i] = make_float4(color.x * phaseS, color.y * phaseS, color.z * phaseS, phaseS);
        so.e0[i] = make_float4(emitted.x, emitted.y, emitted.z, __uint_as_float(newDepth | (dflags & (0x80000000u | CHANNEL_MASK)) | (reqMask << 29)));
        ps.vol_depth[i] = (uint32_t)(vdepth + 1);                           // :378
    }
    for (int o = 16; o > 0; o >>= 1) n_ev += __shfl_down_sync(0xFFFFFFFFu, n_ev, o);
    if ((threadIdx.x & 31) == 0 && n_ev) atomicAdd(&ctr->medium_events, (unsigned long long)n_ev);
}

// parity hook (b200pt_volume_walks): the two volume walks on caller-supplied rays and seeds
__global__ void __launch_bounds__(128) k_volume_walks(DevScene sc, uint32_t n, const float *__restrict__ org, const float *__restrict__ dir, const uint32_t *__restrict__ seeds,
                                                      float ray_depth, float *__restrict__ T_out, float *__restrict__ scatter_out, int32_t *__restrict__ vol_out, uint32_t *__restrict__ rng_out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float3 o = f3(org[3 * i], org[3 * i + 1], org[3 * i + 2]), d = f3(dir[3 * i], dir[3 * i + 1], dir[3 * i + 2]);
    Rng r; r.s = seeds[i];
    T_out[i] = sc.n_grids ? volumes_transmittance_walk(sc, r, o, d, ray_depth) : volumes_transmittance(sc, o, d);
    rng_out[2 * i] = r.s;
    r.s = seeds[i];
    int vi = -1;
    scatter_out[i] = volumes_free_flight(sc, o, d, r, ray_depth, vi);
    vol_out[i] = vi; rng_out[2 * i + 1] = r.s;
}

// ------------------------------------------------------------------------------------------------
// k_prepare_materials : per-material constants of materials whose textures are all 1x1 (DevMaterial::pre0..pre3)
// ------------------------------------------------------------------------------------------------
__global__ void k_prepare_materials(DevMaterial *mats, uint32_t first, uint32_t count) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    DevMaterial &dm = mats[first + j];
    if ((dm.const_mask & 29u) != 29u) { dm.const_mask &= ~32u; return; }     // base, roughness, metallic, emissive textures must all be constant
    Mat m;
    material_load_constants(m, dm.m);
    material_apply_texels(m, dm.cbase, dm.crough, dm.cmetal, dm.cemis);
    dm.pre0 = make_float4(m.BaseColor.x, m.BaseColor.y, m.BaseColor.z, m.Roughness);
    dm.pre1 = make_float4(m.EmissiveColor.x, m.EmissiveColor.y, m.EmissiveColor.z, m.Metallic);
    dm.pre2 = make_float4(m.Ax, m.Ay, m.IOR, 0.0f);
    dm.pre3 = make_float4(m.pm, m.pd, m.pg, 0.0f);
    dm.const_mask |= 32u;
}
void launch_prepare_materials(DevMaterial *mats, uint32_t first, uint32_t count, cudaStream_t st) {
    if (count) k_prepare_materials<<<(count + 127) / 128, 128, 0, st>>>(mats, first, count);
}

// ------------------------------------------------------------------------------------------------
// k_resolve : SH/RayGen.slang:130-159 for every dispatch of the wave, in dispatch order
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_resolve(DevConfig cfg, const DevDispatch *__restrict__ disp, uint32_t n_disp, uint32_t P,
                                                  const float4 *__restrict__ sample_buf, float4 *__restrict__ image) {
    const uint32_t S = cfg.ScreenSplitCount;
    const uint32_t npix = cfg.W * cfg.local_rows;
    const uint32_t LW = (cfg.W + S - 1) / S;
    const float inv_spp = (float)cfg.SampleCount;
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < npix; q += gridDim.x * blockDim.x) {
        float4 px = image[q];
        float3 color = f3(px);
        if (S == 1) {
            for (uint32_t b = 0; b < n_disp; b++) {
                const float3 acc = f3(sample_buf[(size_t)b * P + q]) / inv_spp;                         // :130
                const uint32_t fc = disp[b].FrameCount;
                if (fc > 0) { const float a = 1.0f / (float)(fc + 1u); color = mix3(color, acc, a); }   // :133-137
                else color = acc;
            }
        } else {
            const uint32_t y = q / cfg.W, x = q - y * cfg.W;
            const uint32_t chunk = (x % S) + (y % S) * S;
            const uint32_t sidx = (y / S) * LW + (x / S);
            for (uint32_t b = 0; b < n_disp; b++) {
                const DevDispatch dd = disp[b];
                const float3 acc = f3(sample_buf[(size_t)b * P + sidx]) / inv_spp;
                if (dd.ChunkIndex == chunk) {
                    if (dd.FrameCount > 0) { const float a = 1.0f / (float)(dd.FrameCount + 1u); color = mix3(color, acc, a); }
                    else color = acc;
                } else if (dd.FrameCount == 0 && dd.ChunkIndex == 0) color = acc;                       // splat :144-157
            }
        }
        image[q] = make_float4(color.x, color.y, color.z, 1.0f);
    }
}

// ------------------------------------------------------------------------------------------------
// adaptive sampling (no reference equivalent).  Per local pixel one 16-B record (AdaptivePixel): the running mean and Welford second-moment
// term of the per-frame luminance, the pixel's own frame count n_p and the converged flag.
// ------------------------------------------------------------------------------------------------
// k_resolve_adaptive : k_resolve over the active list.  Entry i of dispatch b (slot b * A + i) belongs to pixel active[i]; the running mean
// uses the pixel's own count n_p in place of FrameCount, which is the same arithmetic for a pixel traced in every frame.
__global__ void __launch_bounds__(256) k_resolve_adaptive(DevConfig cfg, uint32_t n_disp, uint32_t A, const uint32_t *__restrict__ active,
                                                           const float4 *__restrict__ sample_buf, float4 *__restrict__ image, uint4 *__restrict__ state) {
    const float inv_spp = (float)cfg.SampleCount;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < A; i += gridDim.x * blockDim.x) {
        const uint32_t q = active[i];
        const uint4 st = state[q];
        float meanL = __uint_as_float(st.x), M2 = __uint_as_float(st.y);
        uint32_t n = st.z;
        float3 color = f3(image[q]);
        for (uint32_t b = 0; b < n_disp; b++) {
            const float3 acc = f3(sample_buf[(size_t)b * A + i]) / inv_spp;
            if (n > 0) {                                                            // mix3 rounded as k_resolve compiles it: fma(acc, a, color * (1 - a))
                const float a = 1.0f / (float)(n + 1u), ra = 1.0f - a;
                color = f3(__fmaf_rn(acc.x, a, __fmul_rn(color.x, ra)), __fmaf_rn(acc.y, a, __fmul_rn(color.y, ra)), __fmaf_rn(acc.z, a, __fmul_rn(color.z, ra)));
            } else color = acc;
            n++;
            const float L = dot(acc, f3(0.212671f, 0.715160f, 0.072169f));          // the MaxLuminance clamp's weights
            const float delta = L - meanL;                                          // Welford
            meanL += delta / (float)n;
            M2 += delta * (L - meanL);
        }
        image[q] = make_float4(color.x, color.y, color.z, 1.0f);
        state[q] = make_uint4(__float_as_uint(meanL), __float_as_uint(M2), n, st.w);
    }
}

// Relative standard error of the mean luminance with an absolute floor for black pixels: converged iff it is <= Threshold.  Threshold 0 stops
// nothing (a pixel of constant luminance would otherwise meet 0 <= 0).
__device__ __forceinline__ bool adaptive_converged(uint4 st, float threshold, uint32_t min_samples) {
    const uint32_t n = st.z;
    if (threshold <= 0.0f || n < min_samples) return false;
    const float err = sqrtf(__uint_as_float(st.y) / (float)(n - 1u) / (float)n);
    return err <= threshold * fmaxf(__uint_as_float(st.x), 1e-3f);
}

// k_adaptive_update : the decision at an interval boundary (decide == 0: none, the active list is only rebuilt from the flags).  Block t owns
// pixels [t * ADAPTIVE_TILE, (t + 1) * ADAPTIVE_TILE): it flags the pixels that converge and writes how many of its pixels stay active.
__global__ void __launch_bounds__(256) k_adaptive_update(uint4 *__restrict__ state, uint32_t npix, float threshold, uint32_t min_samples, uint32_t decide,
                                                          uint32_t *__restrict__ tile_count) {
    const uint32_t base = blockIdx.x * ADAPTIVE_TILE;
    uint32_t keep = 0;
    for (uint32_t k = threadIdx.x; k < ADAPTIVE_TILE; k += blockDim.x) {
        const uint32_t q = base + k;
        if (q >= npix) break;
        uint4 st = state[q];
        if (!(st.w & PX_CONVERGED) && decide && adaptive_converged(st, threshold, min_samples)) { st.w |= PX_CONVERGED; state[q].w = st.w; }
        keep += (st.w & PX_CONVERGED) ? 0u : 1u;
    }
    keep = __reduce_add_sync(0xFFFFFFFFu, keep);
    __shared__ uint32_t warp_sum[8];
    if ((threadIdx.x & 31u) == 0u) warp_sum[threadIdx.x >> 5] = keep;
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t s = 0; for (uint32_t w = 0; w < blockDim.x / 32u; w++) s += warp_sum[w]; tile_count[blockIdx.x] = s; }
}

// k_adaptive_compact : second pass, stable compaction of the pixels that stay active into the active list (pixel order, so neighbouring pixels
// keep neighbouring lanes and their camera rays stay coherent).  A tile's offset is the sum of the counts of the tiles before it; inside the
// tile, 256 pixels per round are placed by a warp ballot / popc and a scan over the 8 warp counts.  The last block writes the active count A.
__global__ void __launch_bounds__(256) k_adaptive_compact(const uint4 *__restrict__ state, uint32_t npix, const uint32_t *__restrict__ tile_count,
                                                           uint32_t *__restrict__ active, uint32_t *__restrict__ active_count) {
    __shared__ uint32_t warp_sum[8], s_base;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t part = 0;
    for (uint32_t t = threadIdx.x; t < blockIdx.x; t += blockDim.x) part += tile_count[t];
    part = __reduce_add_sync(0xFFFFFFFFu, part);
    if (lane == 0u) warp_sum[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t s = 0; for (uint32_t w = 0; w < 8u; w++) s += warp_sum[w]; s_base = s; }
    __syncthreads();
    uint32_t base = s_base;
    for (uint32_t r = 0; r < ADAPTIVE_TILE / 256u; r++) {
        const uint32_t q = blockIdx.x * ADAPTIVE_TILE + r * 256u + threadIdx.x;
        const bool keep = q < npix && !(state[q].w & PX_CONVERGED);
        const uint32_t bal = __ballot_sync(0xFFFFFFFFu, keep);
        __syncthreads();                                                    // warp_sum of the previous round has been read
        if (lane == 0u) warp_sum[warp] = (uint32_t)__popc(bal);
        __syncthreads();
        uint32_t before = 0, total = 0;
        #pragma unroll
        for (uint32_t w = 0; w < 8u; w++) { const uint32_t c = warp_sum[w]; before += w < warp ? c : 0u; total += c; }
        if (keep) active[base + before + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = q;
        base += total;
    }
    if (blockIdx.x == gridDim.x - 1u && threadIdx.x == 0) *active_count = base;
}

// ------------------------------------------------------------------------------------------------
// kernel selectors: the instantiation each launch runs for its flags.  The launchers launch through them, and query_launch_cfg sizes the
// grids of, checks big mode against and opts in the shared memory of exactly what they can return.
// ------------------------------------------------------------------------------------------------
static auto extend_kernel(bool smem, bool primary, bool uniform) {
    const decltype(&k_extend<false, false, false>) fn[2][2][2] = {
        { { k_extend<false, false, false>, k_extend<false, false, true> }, { k_extend<false, true, false>, k_extend<false, true, true> } },
        { { k_extend<true, false, false>, k_extend<true, false, true> }, { k_extend<true, true, false>, k_extend<true, true, true> } } };
    return fn[smem][primary][uniform];
}
static auto extend_dyn_kernel(bool smem, bool primary, bool wide) {        // the BVH4 is never staged in shared memory
    if (wide) return primary ? k_extend_dyn<false, true, true> : k_extend_dyn<false, false, true>;
    if (smem) return primary ? k_extend_dyn<true, true, false> : k_extend_dyn<true, false, false>;
    return primary ? k_extend_dyn<false, true, false> : k_extend_dyn<false, false, false>;
}
static auto shadow_dyn_kernel(bool smem, bool wide) {
    return wide ? k_shadow_dyn<false, true> : (smem ? k_shadow_dyn<true, false> : k_shadow_dyn<false, false>);
}
static auto camera_kernel(bool uniform, bool adaptive) {
    return uniform ? (adaptive ? k_camera<true, true> : k_camera<true, false>) : (adaptive ? k_camera<false, true> : k_camera<false, false>);
}
static auto shade_kernel(uint32_t cls, bool vol, bool fuse) {              // the fused kernels run only without a pre-pass
    const decltype(&k_shade_hit<MC_GENERAL, false, false>) fn[MC_COUNT][3] = {
        { k_shade_hit<MC_DIFFUSE, false, false>, k_shade_hit<MC_DIFFUSE, true, false>, k_shade_hit<MC_DIFFUSE, false, true> },
        { k_shade_hit<MC_METAL, false, false>, k_shade_hit<MC_METAL, true, false>, k_shade_hit<MC_METAL, false, true> },
        { k_shade_hit<MC_GLASS, false, false>, k_shade_hit<MC_GLASS, true, false>, k_shade_hit<MC_GLASS, false, true> },
        { k_shade_hit<MC_GENERAL, false, false>, k_shade_hit<MC_GENERAL, true, false>, k_shade_hit<MC_GENERAL, false, true> } };
    return fn[cls][fuse ? 2 : (int)vol];
}
static auto connect_kernel(bool smem, bool trace, bool walks) {            // without tracing (behind k_shadow_dyn) the BVH is not read
    if (!trace) return walks ? k_connect<false, false, true> : k_connect<false, false, false>;
    if (smem) return walks ? k_connect<true, true, true> : k_connect<true, true, false>;
    return walks ? k_connect<false, true, true> : k_connect<false, true, false>;
}
static auto volume_decide_kernel(bool smem) { return smem ? k_volume_decide<true> : k_volume_decide<false>; }

// ------------------------------------------------------------------------------------------------
// launch configuration
// ------------------------------------------------------------------------------------------------
static constexpr size_t DYN_RING_BYTES_HOST = 8 * 128 * sizeof(uint32_t);
static size_t trace_smem_bytes(const DevScene &sc, int max_stack, int threads, bool smem) {
    return (size_t)max_stack * threads * sizeof(int) + (smem ? sc.bvh_bytes : 0);
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) applies to the CURRENT device only, and the C-ABI lets one process drive several GPUs
// (b200pt_create(device, ..)): the opt-in is tracked per device ordinal.  It covers every flag combination of every selector.
static unsigned long long g_attr_done_mask = 0ull;
static int opt_in_shared_memory() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return (int)cudaGetLastError();
    if (dev >= 0 && dev < 64 && ((g_attr_done_mask >> dev) & 1ull)) return 0;
    // the 227 KB per-CTA limit covers static + dynamic, so each kernel gets 227 KB minus its static part
    int rc = 0;
    auto optin = [&rc](auto f) {
        cudaFuncAttributes a{};
        cudaError_t e = cudaFuncGetAttributes(&a, f);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - (int)a.sharedSizeBytes);
        if (e != cudaSuccess && rc == 0) rc = (int)e;
    };
    for (int f = 0; f < 8; f++) {
        const bool a = f & 1, b = f & 2, c = f & 4;
        optin(extend_kernel(a, b, c)); optin(extend_dyn_kernel(a, b, c)); optin(connect_kernel(a, b, c));
        optin(shadow_dyn_kernel(a, b)); optin(camera_kernel(a, b));
        optin(volume_decide_kernel(a)); optin(features_kernel(a));
        for (uint32_t cls = 0; cls < MC_COUNT; cls++) optin(shade_kernel(cls, a, b));
    }
    cudaGetLastError();
    if (rc == 0 && dev >= 0 && dev < 64) g_attr_done_mask |= 1ull << dev;
    return rc;
}

int bvh4_stack_entries(int bvh4_depth, int cap) {
    const int need = 3 * bvh4_depth + 2;                                    // worst case: three pushes per level
    const int entries = need < cap ? need : cap;
    return need - entries > DYN_SPILL ? 0 : entries;
}

// grid sizing: persistent grids = SM count x resident CTAs per SM for the chosen shared-memory footprint
int query_launch_cfg(const DevScene &sc, int bvh_max_depth, int bvh4_depth, LaunchCfg *lc) {
    { const int a = opt_in_shared_memory(); if (a != 0) return a; }
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceProp prop; cudaError_t e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return (int)e;
    const int sms = prop.multiProcessorCount;
    // depth + 2 entries always suffice for the near-first walk (one push per level).  A full stack would drop the push -- a lost subtree, i.e.
    // wrong hits with no error -- so a tree deeper than lbvh_refine_sah normally leaves (BVH_STACK_MAX) gets a deeper stack, and the scene is
    // refused below when the shared memory of a launch cannot hold it.
    lc->max_stack = std::max(bvh_max_depth + 2, 4);
    // Whole BVH in shared memory: <= 64 KiB -> several CTAs per SM (Cornell: 1.3 KiB); up to what fits beside the stacks of ONE 512-thread CTA per SM
    // -> "big" mode (config 4's glass scene: 108 KiB): k_extend, k_connect, k_camera and the fused k_shade_hit run 512-thread CTAs.
    const bool aligned = sc.bvh_bytes > 0 && (sc.bvh_bytes % 16u) == 0;
    const bool fits_small = aligned && sc.bvh_bytes <= 64u * 1024u;
    // Big mode runs the one-ray-per-thread kernels over the shared-memory BVH at 8-16 warps per SM with divergent LDS; the dynamic-fetch kernels
    // over L2 are the default there -> big mode is OPT-IN (B200PT_SMEM_BIG=1).  Each of those 512-thread kernels must fit the stacks and the BVH
    // into its opt-in limit: 227 KiB minus its static shared memory (k_camera's flat-walk table, ~4 KiB, is the largest).
    bool fits_big = false;
    if (const char *e = getenv("B200PT_SMEM_BIG")) {
        if (atoi(e) == 1 && aligned && !fits_small) {
            const size_t need = trace_smem_bytes(sc, lc->max_stack, 512, true);
            fits_big = true;
            auto fits = [&](auto f) { cudaFuncAttributes a{}; if (cudaFuncGetAttributes(&a, f) != cudaSuccess || need + a.sharedSizeBytes > 227u * 1024u) fits_big = false; };
            for (int f = 0; f < 4; f++) {                                   // f: two flags, or the material class
                const bool a = f & 1, b = f & 2;
                fits(extend_kernel(true, a, b)); fits(camera_kernel(a, b)); fits(connect_kernel(true, true, a)); fits(shade_kernel(f, false, true));
            }
        }
    }
    lc->bvh_in_smem = fits_small || fits_big;
    lc->big = fits_big;
    const bool smem = lc->bvh_in_smem;
    // traversal shape: dynamic-fetch while-while kernels (bvh_dynfetch.cuh) over the BVH4 when the BVH lives in L2/HBM, one ray per thread
    // over the BVH2 when the whole BVH sits in shared memory (tiny scenes: no divergence or latency to recover).
    // Overrides: B200PT_TRAV=classic|dyn, B200PT_WIDE=0|1, B200PT_DYN_THRESH=1..32, B200PT_WIDE_STACK=<shared-memory stack entries>.
    lc->trav_dyn = !smem;
    if (const char *e = getenv("B200PT_TRAV")) { if (!strcmp(e, "dyn")) lc->trav_dyn = true; else if (!strcmp(e, "classic")) lc->trav_dyn = false; }
    lc->dyn_thresh = 20;
    if (const char *e = getenv("B200PT_DYN_THRESH")) { int v = atoi(e); if (v >= 1 && v <= 32) lc->dyn_thresh = v; }
    lc->wide = lc->trav_dyn && !smem && sc.nodes4 != nullptr && sc.bvh_bytes >= (8u << 20);   // small BVHs stay L1/L2-hot: BVH2 is cheaper there
    if (const char *e = getenv("B200PT_WIDE")) { if (atoi(e) == 1 && lc->trav_dyn && !smem && sc.nodes4 != nullptr) lc->wide = true; }
    if (const char *e = getenv("B200PT_WIDE")) { if (atoi(e) == 0) lc->wide = false; }
    lc->dyn_stack = lc->max_stack;                                          // BVH2: depth + 2 entries always suffice
    lc->wide_cap = WIDE_STACK_DEFAULT;
    if (const char *e = getenv("B200PT_WIDE_STACK")) { int v = atoi(e); if (v >= 4 && v <= 96) lc->wide_cap = v; }
    if (lc->wide) {
        lc->dyn_stack = bvh4_stack_entries(bvh4_depth, lc->wide_cap);
        if (lc->dyn_stack == 0) lc->wide = false, lc->dyn_stack = lc->max_stack;   // deeper than shared column + overflow array: BVH2
    }
    // Bounce pipeline of scenes whose BVH is staged in shared memory and walked one ray per thread (the default elsewhere is 0):
    //   1 (default): k_shade_hit<., ., true> traces each NEE query the moment it is built and finishes the path (roulette, radiance, compaction)
    //      in the same thread; the next segment's closest hit runs in k_extend<true, false, .>.
    // B200PT_FUSE=0 overrides (k_extend + k_shade_hit + k_connect); any other value keeps the default.
    lc->fuse = (smem && !lc->trav_dyn) ? 1 : 0;
    if (const char *e = getenv("B200PT_FUSE")) { const int v = atoi(e); if ((v == 0 || v == 1) && smem && !lc->trav_dyn) lc->fuse = v; }
    // Camera rays of those scenes: generated and traced in one kernel (k_camera) instead of k_raygen + k_extend<true, true, .>, unless the scene
    // needs a pre-pass (decided per call: plan_call).  B200PT_CAMERA=0 keeps the pair.
    lc->camera = smem && !lc->trav_dyn;
    if (const char *e = getenv("B200PT_CAMERA")) { if (atoi(e) == 0) lc->camera = false; }

    // CTA sizes and dynamic shared memory of each launch shape; the dynamic-fetch kernels always run 256-thread CTAs
    lc->extend_threads = fits_big && !lc->trav_dyn ? 512 : 256;
    lc->bounce_threads = fits_big ? 512 : 128;
    lc->smem_extend = trace_smem_bytes(sc, lc->trav_dyn ? lc->dyn_stack + 1 : lc->max_stack, lc->extend_threads, smem);
    lc->smem_shadow = trace_smem_bytes(sc, lc->dyn_stack + 1, 256, smem) + DYN_RING_BYTES_HOST;
    lc->smem_bounce = trace_smem_bytes(sc, lc->max_stack, lc->bounce_threads, true);
    lc->smem_trace = trace_smem_bytes(sc, lc->max_stack, 256, smem);
    // A stack the launches cannot hold (a tree far deeper than BVH_STACK_MAX): refuse the scene rather than truncate.  Big mode was checked
    // against each kernel's own static shared memory above; elsewhere 8 KiB bounds it (k_camera's flat-walk table, ~4 KiB, is the largest).
    if (!fits_big)
        for (const size_t b : { lc->smem_extend, lc->smem_shadow, smem ? lc->smem_bounce : 0u, lc->smem_trace })   // the fused k_shade_hit runs only over a staged BVH
            if (b + 8u * 1024u > 227u * 1024u) return (int)cudaErrorInvalidConfiguration;
    auto occupancy = [](auto fn, int threads, size_t smem_bytes) { int n = 0; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, threads, smem_bytes); return n; };
    int occ_e = 0, occ_c = 0, occ_sh = 0;
    if (lc->trav_dyn) {
        occ_e = occupancy(extend_dyn_kernel(smem, false, lc->wide), lc->extend_threads, lc->smem_extend);
        occ_sh = occupancy(shadow_dyn_kernel(smem, lc->wide), 256, lc->smem_shadow);
        occ_c = occupancy(connect_kernel(smem, false, false), lc->extend_threads, 0);
    } else {
        occ_e = occupancy(extend_kernel(smem, false, false), lc->extend_threads, lc->smem_extend);
        if (smem) occ_e = std::min(occ_e, occupancy(extend_kernel(true, false, true), lc->extend_threads, lc->smem_extend));   // one grid for both tally forms: the smaller residency
        occ_c = occupancy(connect_kernel(smem, true, false), lc->extend_threads, lc->smem_extend);
    }
    // every unfused k_shade_hit runs on the grid of the general one, every fused one on the grid of the fused general one
    const int occ_s = std::max(1, occupancy(shade_kernel(MC_GENERAL, false, false), 128, 0));
    const int occ_b = std::max(1, smem ? occupancy(shade_kernel(MC_GENERAL, false, true), lc->bounce_threads, lc->smem_bounce) : 0);
    int occ_cam = 0;                                                        // both camera forms on one grid: the smaller residency
    if (lc->camera) occ_cam = std::min(occupancy(camera_kernel(false, false), lc->extend_threads, lc->smem_extend),
                                       occupancy(camera_kernel(true, false), lc->extend_threads, lc->smem_extend));
    occ_e = std::max(1, occ_e); occ_c = std::max(1, occ_c); occ_sh = std::max(1, occ_sh);
    lc->grid_extend = sms * occ_e; lc->grid_connect = sms * occ_c; lc->grid_shadow = sms * occ_sh;
    lc->grid_shade = sms * occ_s;
    lc->grid_bounce = sms * occ_b;
    lc->grid_camera = sms * std::max(1, occ_cam);
    lc->grid_volume_decide = sms * std::max(1, occupancy(volume_decide_kernel(smem), 256, lc->smem_trace));
    lc->grid_features = sms * std::max(1, occupancy(features_kernel(smem), 256, lc->smem_trace));
    lc->grid_light = sms * 8;
    if (getenv("B200PT_DEBUG"))
        fprintf(stderr, "[b200pt] launch cfg: bvh depth %d (bvh4 %d) max_stack %d dyn_stack %d bvh_bytes %u smem %d dyn %d wide %d thresh %d fuse %d big %d camera %d | CTAs/SM extend %d connect %d shadow %d shade %d bounce %d camera %d\n",
                bvh_max_depth, bvh4_depth, lc->max_stack, lc->dyn_stack, sc.bvh_bytes, (int)smem, (int)lc->trav_dyn, (int)lc->wide, lc->dyn_thresh, lc->fuse, (int)lc->big, (int)lc->camera,
                occ_e, occ_c, occ_sh, occ_s, occ_b, occ_cam);
    return 0;
}

CallPlan plan_call(const LaunchCfg &lc, const DevScene &sc, const DevConfig &cfg, bool medium, uint32_t class_mask) {
    CallPlan cp;
    cp.pre = sc.n_volumes != 0u || cfg.EnableAtmosphere != 0u;              // volumes and / or the atmosphere (csrc/atmosphere.cuh)
    cp.fuse = lc.fuse != 0 && !cp.pre;                                      // the fused shading kernels need the BVH in shared memory and no volumes
    cp.camera = lc.camera && !cp.pre;
    cp.uniform = sc.uniform_class != 0xFFu && !cp.pre;
    cp.walks = cfg.EnableAtmosphere != 0u || sc.n_grids != 0u;
    cp.class_mask = cp.pre ? (class_mask | (1u << MC_GENERAL)) : class_mask;   // volume / atmosphere events ride in the general queue
    // WAVE_IMPLIED: k_camera's paths are all inside the image only without chunked dispatch (overhang paths are born dead and keep their full
    // state), and only the fused shading kernels infer the state.  WAVE_STORE: sub-wave 0 ends every path exactly once when the bounce loop
    // provably runs dry -- not with a pre-pass (DEAD_EVENT ends, channel-split paths), not with medium walks (the runaway guard may stop them),
    // not at MaxDepth 0 (no bounce runs, the slots must read zero).
    cp.implied = cp.camera && cfg.ScreenSplitCount == 1u && cp.fuse;
    cp.store = !cp.pre && !medium && cfg.MaxDepth > 0u;
    return cp;
}

// ------------------------------------------------------------------------------------------------
// host-callable launchers
// ------------------------------------------------------------------------------------------------
int launch_raygen(const LaunchCfg &lc, const DevConfig &cfg, const DevDispatch *disp, uint32_t n_disp, uint32_t P, uint32_t first_sample, uint32_t flags,
                  const uint32_t *rng_carry, PathState ps, float4 *sample_buf, uint32_t *ctrl, WaveCounters *ctr, cudaStream_t st, const uint32_t *active) {
    if (active) k_raygen<true><<<lc.grid_light, 256, 0, st>>>(cfg, disp, n_disp, P, first_sample, flags, rng_carry, ps, sample_buf, ctrl, ctr, active);
    else k_raygen<false><<<lc.grid_light, 256, 0, st>>>(cfg, disp, n_disp, P, first_sample, flags, rng_carry, ps, sample_buf, ctrl, ctr, nullptr);
    return 1;
}
int launch_camera(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, const DevConfig &cfg, const DevDispatch *disp, uint32_t n_disp, uint32_t P,
                  uint32_t first_sample, uint32_t flags, const uint32_t *rng_carry, PathState ps, float4 *sample_buf, float4 *hit_out, uint32_t *ctrl, Queues q,
                  WaveCounters *ctr, cudaStream_t st, const uint32_t *active) {
    camera_kernel(cp.uniform, active != nullptr)<<<lc.grid_camera, lc.extend_threads, lc.smem_extend, st>>>(sc, cfg, disp, n_disp, P, first_sample, flags, rng_carry, ps,
                                                                                                           sample_buf, hit_out, ctrl, q, lc.max_stack, ctr, active);
    return 1;
}
void launch_resolve_adaptive(const LaunchCfg &lc, const DevConfig &cfg, uint32_t n_disp, uint32_t A, const uint32_t *active,
                             const float4 *sample_buf, float4 *image, uint4 *state, cudaStream_t st) {
    k_resolve_adaptive<<<lc.grid_light, 256, 0, st>>>(cfg, n_disp, A, active, sample_buf, image, state);
}
void launch_adaptive_update(uint4 *state, uint32_t npix, float threshold, uint32_t min_samples, bool decide, uint32_t *tile_count,
                            uint32_t *active, uint32_t *active_count, cudaStream_t st) {
    const uint32_t tiles = (npix + ADAPTIVE_TILE - 1u) / ADAPTIVE_TILE;
    if (!tiles) { cudaMemsetAsync(active_count, 0, sizeof(uint32_t), st); return; }
    k_adaptive_update<<<tiles, 256, 0, st>>>(state, npix, threshold, min_samples, decide ? 1u : 0u, tile_count);
    k_adaptive_compact<<<tiles, 256, 0, st>>>(state, npix, tile_count, active, active_count);
}
int launch_extend(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, PathState ps, float4 *hit_out, uint32_t *ctrl, uint32_t parity, Queues q,
                  WaveCounters *ctr, bool primary, cudaStream_t st) {
    if (lc.trav_dyn)
        extend_dyn_kernel(lc.bvh_in_smem, primary, lc.wide)<<<lc.grid_extend, lc.extend_threads, lc.smem_extend, st>>>(sc, ps, hit_out, ctrl, parity, q, lc.dyn_stack, lc.dyn_thresh, ctr);
    else extend_kernel(lc.bvh_in_smem, primary, cp.uniform)<<<lc.grid_extend, lc.extend_threads, lc.smem_extend, st>>>(sc, ps, hit_out, ctrl, parity, q, lc.max_stack, ctr);
    return 1;
}
// k_shade_miss + one k_shade_hit<CLASS> per material class of the call (+ k_shade_volume).  cp.fuse: see k_shade_hit.
int launch_shade(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, const DevConfig &cfg, PathState ps, PathState dst, ShadeOut so, const float4 *hit_in,
                 uint32_t *ctrl, uint32_t parity, Queues q, float4 *sample_buf, uint32_t *rng_carry, WaveCounters *ctr, uint32_t flags, cudaStream_t st) {
    int launched = 1;
    k_shade_miss<<<lc.grid_light, 256, 0, st>>>(sc, cfg, ps, ctrl, parity, q.miss, sample_buf, rng_carry, ctr, flags);
    for (uint32_t c = 0; c < MC_COUNT; c++) {
        if (!(cp.class_mask & (1u << c))) continue;
        launched++;
        shade_kernel(c, cp.pre, cp.fuse)<<<cp.fuse ? lc.grid_bounce : lc.grid_shade, cp.fuse ? lc.bounce_threads : 128, cp.fuse ? lc.smem_bounce : 0, st>>>(
            sc, cfg, ps, dst, so, hit_in, ctrl, parity, q, sample_buf, rng_carry, lc.max_stack, ctr, flags);
    }
    if (cp.pre) { launched++; k_shade_volume<<<lc.grid_light, 128, 0, st>>>(sc, cfg, ps, so, ctrl, parity, q, ctr); }
    return launched;
}
int launch_volume_decide(const LaunchCfg &lc, const DevScene &sc, const DevConfig &cfg, PathState ps, ShadeOut so, const uint32_t *ctrl, uint32_t parity,
                         float4 *sample_buf, uint32_t *rng_carry, cudaStream_t st) {
    volume_decide_kernel(lc.bvh_in_smem)<<<lc.grid_volume_decide, 256, lc.smem_trace, st>>>(sc, cfg, ps, so, ctrl, parity, lc.max_stack, sample_buf, rng_carry);
    return 1;
}
int launch_connect(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, const DevConfig &cfg, PathState src, PathState dst, ShadeOut so,
                   uint32_t *ctrl, uint32_t parity, Queues q, float4 *sample_buf, uint32_t *rng_carry, WaveCounters *ctr, uint32_t flags, cudaStream_t st) {
    int launched = 1;
    if (lc.trav_dyn) {                                                      // shadow rays in their own dynamic-fetch kernel, then the join without tracing
        shadow_dyn_kernel(lc.bvh_in_smem, lc.wide)<<<lc.grid_shadow, 256, lc.smem_shadow, st>>>(sc, so, ctrl, parity, q, lc.dyn_stack, lc.dyn_thresh, ctr);
        launched++;
    }
    connect_kernel(lc.bvh_in_smem, !lc.trav_dyn, cp.walks)<<<lc.grid_connect, lc.extend_threads, lc.trav_dyn ? 0 : lc.smem_extend, st>>>(
        sc, cfg, src, dst, so, ctrl, parity, q, sample_buf, rng_carry, lc.max_stack, ctr, flags);
    return launched;
}
void launch_resolve(const LaunchCfg &lc, const DevConfig &cfg, const DevDispatch *disp, uint32_t n_disp, uint32_t P,
                    const float4 *sample_buf, float4 *image, cudaStream_t st) {
    k_resolve<<<lc.grid_light, 256, 0, st>>>(cfg, disp, n_disp, P, sample_buf, image);
}
void launch_volume_walks(const DevScene &sc, uint32_t n, const float *org, const float *dir, const uint32_t *seeds, float ray_depth,
                         float *T_out, float *scatter_out, int32_t *vol_out, uint32_t *rng_out, cudaStream_t st) {
    k_volume_walks<<<(n + 127u) / 128u, 128, 0, st>>>(sc, n, org, dir, seeds, ray_depth, T_out, scatter_out, vol_out, rng_out);
}

} // namespace b200pt
