// denoise_kernels.cu -- the denoiser of the accumulated image (sm_90a, no reference equivalent).
//
//   k_features        albedo / coverage / normal / view depth of the first surface seen through each pixel (FeatureSamples camera rays)
//   k_record_variance variance of each pixel's mean luminance from the Welford records of k_resolve_adaptive
//   k_dn_prepare      demodulation by the albedo, variance demodulation, depth gradient
//   k_dn_atrous       one pass of the a-trous wavelet filter (Dammertz et al. 2010) with the SVGF edge-stopping weights (Schied et al. 2017)
//   k_dn_remodulate   multiplication by the albedo
//
// Kept out of wavefront_kernels.cu so that every kernel of the render path keeps its code.  DESIGN.md section 12 states the filter; the
// float64 model in tests/test_denoiser.py restates it.
#include "bvh_traverse.cuh"
#include "camera.cuh"
#include "kernels.h"

namespace b200pt {

// ------------------------------------------------------------------------------------------------
// k_features : FeatureSamples camera rays per local pixel from one PCG stream seeded y + W * x + seed0 (global pixel coordinates, so a tile
// partition's rows equal the one-rank rows), each drawing its jitter and lens samples in camera_ray's order.  The closest hit of each ray
// (the walk of b200pt_trace_closest after k_extend's normalize_ray) gives albedo (pd + pm) * BaseColor + pg, the shading normal and the view depth;
// a miss counts as albedo 1, normal 0.  Volumes and the atmosphere are not seen: the features are those of the first surface.
// ------------------------------------------------------------------------------------------------
template <bool SMEM>
__global__ void __launch_bounds__(256) k_features(DevScene sc, DevConfig cfg, float3 fwd, uint32_t samples, uint32_t seed0, int max_stack,
                                                  float4 *__restrict__ albedo_cov, float4 *__restrict__ normal_depth) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar;
    int *stack = reinterpret_cast<int *>(smem) + threadIdx.x;
    BvhView bv;
    if (SMEM) bv = stage_bvh_smem(sc, smem + (size_t)max_stack * blockDim.x * sizeof(int), &bar);
    else bv = global_bvh(sc);
    const uint32_t npix = cfg.W * cfg.local_rows;
    const float3 eye = camera_eye(cfg);
    const float inv_n = 1.0f / (float)samples;
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < npix; q += gridDim.x * blockDim.x) {
        const uint32_t lr = q / cfg.W, x = q - lr * cfg.W;
        const uint32_t y = part_global_row(lr, cfg.rank, cfg.world, cfg.band_rows);
        Rng rng; rng.s = y + cfg.W * x + seed0;
        float3 alb = f3(0.0f), nrm = f3(0.0f);
        float z = 0.0f; uint32_t hits = 0;
        for (uint32_t s = 0; s < samples; s++) {
            float3 o, d;
            camera_ray(cfg, x, y, rng, o, d);
            const float3 rd = normalize_ray(d);
            HitRec h;
            if (!bvh_trace<SMEM, false>(bv, o, rd, 0.01f, 100000.0f, h, stack, (int)blockDim.x, max_stack)) { alb = alb + f3(1.0f); continue; }
            float4 g[7];
            const float4 *gp = reinterpret_cast<const float4 *>(sc.shade_tris + h.gid);
            #pragma unroll
            for (int k = 0; k < 7; k++) g[k] = __ldg(gp + k);
            const DevInstance &in = sc.instances[__float_as_uint(g[0].w)];
            const DevMaterial &cm = sc.materials[__float_as_uint(g[2].w)];
            Surface sf;
            surface_init(sf, sc, cfg, in, g, h.u, h.v, rd, cm);
            Mat m;
            material_init(m, sc, cfg, cm, sf);
            alb = alb + (m.BaseColor * (m.pd + m.pm) + f3(m.pg));
            nrm = nrm + sf.Normal;
            z += dot(sf.WorldPos - eye, fwd);
            hits++;
        }
        albedo_cov[q] = make_float4(alb.x * inv_n, alb.y * inv_n, alb.z * inv_n, (float)hits * inv_n);
        normal_depth[q] = make_float4(nrm.x * inv_n, nrm.y * inv_n, nrm.z * inv_n, hits ? z / (float)hits : 0.0f);
    }
}

// variance of the mean luminance M2 / (n - 1) / n of each record (kernels.h: {meanL, M2, n_p, flags}); DN_UNKNOWN_VARIANCE below two frames
__global__ void __launch_bounds__(256) k_record_variance(const uint4 *__restrict__ state, uint32_t npix, float *__restrict__ var) {
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < npix; q += gridDim.x * blockDim.x) {
        const uint4 st = state[q];
        var[q] = st.z < 2u ? DN_UNKNOWN_VARIANCE : __uint_as_float(st.y) / (float)(st.z - 1u) / (float)st.z;
    }
}

__device__ __forceinline__ float dn_lum(float x, float y, float z) { return 0.212671f * x + 0.715160f * y + 0.072169f * z; }   // the MaxLuminance clamp's weights

// Demodulation: iv = (c / max(a, 1e-3), v / max(lum(a), 1e-3)^2).  aux = (dz/dx, dz/dy, coverage, 0): central differences of the feature
// depth, one-sided at the image border and next to pixels with coverage 0, 0 where neither neighbour is usable.
__global__ void __launch_bounds__(256) k_dn_prepare(uint32_t W, uint32_t H, const float4 *__restrict__ color, const float4 *__restrict__ albedo_cov,
                                                    const float4 *__restrict__ normal_depth, const float *__restrict__ variance,
                                                    float4 *__restrict__ iv, float4 *__restrict__ aux) {
    const uint32_t npix = W * H;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
        const uint32_t y = p / W, x = p - y * W;
        const float4 c = color[p], a = albedo_cov[p];
        const float ax = fmaxf(a.x, 1e-3f), ay = fmaxf(a.y, 1e-3f), az = fmaxf(a.z, 1e-3f);
        const float la = fmaxf(dn_lum(a.x, a.y, a.z), 1e-3f);
        iv[p] = make_float4(c.x / ax, c.y / ay, c.z / az, variance[p] / (la * la));
        const float zc = normal_depth[p].w;
        auto grad = [&](bool lo_in, uint32_t lo, bool hi_in, uint32_t hi) {
            const bool l = lo_in && albedo_cov[lo].w > 0.0f, h = hi_in && albedo_cov[hi].w > 0.0f;
            if (l && h) return 0.5f * (normal_depth[hi].w - normal_depth[lo].w);
            if (h) return normal_depth[hi].w - zc;
            if (l) return zc - normal_depth[lo].w;
            return 0.0f;
        };
        const float gx = grad(x > 0, p - 1, x + 1 < W, p + 1), gy = grad(y > 0, p - W, y + 1 < H, p + W);
        aux[p] = make_float4(gx, gy, a.w, 0.0f);
    }
}

// One a-trous pass with step s: 5x5 B3-spline taps at offsets s * {-2..2} (taps outside the image are dropped), weight
// h * w_l * w_n * w_z (w_n = w_z = 1 between two pixels without coverage, w = 0 between a covered and an uncovered one).
// w_l uses the standard deviation of a normalised 3x3 Gaussian of the current variance around p.
__global__ void __launch_bounds__(256) k_dn_atrous(uint32_t W, uint32_t H, uint32_t s, const float4 *__restrict__ iv_in, const float4 *__restrict__ normal_depth,
                                                   const float4 *__restrict__ aux, float sigma_l, float sigma_n, float sigma_z, float4 *__restrict__ iv_out) {
    const float hk[5] = { 1.0f / 16.0f, 1.0f / 4.0f, 3.0f / 8.0f, 1.0f / 4.0f, 1.0f / 16.0f };
    const float gk[3] = { 0.25f, 0.5f, 0.25f };
    const uint32_t npix = W * H;
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
        const int y = (int)(p / W), x = (int)(p - (uint32_t)y * W);
        const float4 cp = iv_in[p];
        float gs = 0.0f, gw = 0.0f;
        #pragma unroll
        for (int j = -1; j <= 1; j++) {
            if (y + j < 0 || y + j >= (int)H) continue;
            #pragma unroll
            for (int i = -1; i <= 1; i++) {
                if (x + i < 0 || x + i >= (int)W) continue;
                const float g = gk[i + 1] * gk[j + 1];
                gs += g * iv_in[(size_t)(y + j) * W + (uint32_t)(x + i)].w; gw += g;
            }
        }
        const float lp = dn_lum(cp.x, cp.y, cp.z);
        const float den_l = sigma_l * sqrtf(gs / gw) + 1e-6f;
        const float4 np = normal_depth[p], ap = aux[p];
        const bool covp = ap.z > 0.0f;
        const float zfloor = 1e-3f * fmaxf(np.w, 1e-3f);
        float sw = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f, sv = 0.0f;
        #pragma unroll
        for (int j = -2; j <= 2; j++) {
            const int qy = y + j * (int)s;
            if (qy < 0 || qy >= (int)H) continue;
            #pragma unroll
            for (int i = -2; i <= 2; i++) {
                const int qx = x + i * (int)s;
                if (qx < 0 || qx >= (int)W) continue;
                const size_t q = (size_t)qy * W + (uint32_t)qx;
                const bool covq = aux[q].z > 0.0f;
                if (covp != covq) continue;
                const float4 cq = iv_in[q];
                float w = hk[i + 2] * hk[j + 2] * expf(-fabsf(lp - dn_lum(cq.x, cq.y, cq.z)) / den_l);
                if (covp) {
                    const float4 nq = normal_depth[q];
                    const float wn = powf(fmaxf(0.0f, np.x * nq.x + np.y * nq.y + np.z * nq.z), sigma_n);
                    const float dz = fabsf(ap.x * (float)(i * (int)s) + ap.y * (float)(j * (int)s));
                    w *= wn * expf(-fabsf(np.w - nq.w) / (sigma_z * dz + zfloor));
                }
                if (!(w > 0.0f)) continue;
                sw += w; sr += w * cq.x; sg += w * cq.y; sb += w * cq.z;
                const float w2 = w * w;
                if (w2 > 0.0f) sv += w2 * cq.w;
            }
        }
        iv_out[p] = sw > 0.0f ? make_float4(sr / sw, sg / sw, sb / sw, sv / sw / sw) : cp;
    }
}

__global__ void __launch_bounds__(256) k_dn_remodulate(uint32_t npix, const float4 *__restrict__ iv, const float4 *__restrict__ albedo_cov,
                                                       const float4 *__restrict__ color, float4 *__restrict__ out) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
        const float4 v = iv[p], a = albedo_cov[p];
        out[p] = make_float4(v.x * fmaxf(a.x, 1e-3f), v.y * fmaxf(a.y, 1e-3f), v.z * fmaxf(a.z, 1e-3f), color[p].w);
    }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
static int streaming_grid(uint32_t n) {
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const uint32_t blocks = (n + 255u) / 256u, cap = (uint32_t)sms * 8u;
    return (int)(blocks < 1u ? 1u : (blocks < cap ? blocks : cap));
}

FeaturesKernel features_kernel(bool smem) { return smem ? k_features<true> : k_features<false>; }

int launch_features(const LaunchCfg &lc, const DevScene &sc, const DevConfig &cfg, float3 forward, uint32_t samples, uint32_t seed0,
                    float4 *albedo_cov, float4 *normal_depth, cudaStream_t st) {
    // persistent grid (query_launch_cfg): each CTA stages the BVH once
    features_kernel(lc.bvh_in_smem)<<<lc.grid_features, 256, lc.smem_trace, st>>>(sc, cfg, forward, samples, seed0, lc.max_stack, albedo_cov, normal_depth);
    return (int)cudaGetLastError();
}

void launch_record_variance(const uint4 *state, uint32_t npix, float *variance, cudaStream_t st) {
    k_record_variance<<<streaming_grid(npix), 256, 0, st>>>(state, npix, variance);
}

void launch_denoise_filter(uint32_t W, uint32_t H, const float4 *color, const float4 *albedo_cov, const float4 *normal_depth, const float *variance,
                           uint32_t iterations, float sigma_l, float sigma_n, float sigma_z, float4 *scratch, float4 *out, cudaStream_t st) {
    const uint32_t npix = W * H;
    if (!npix) return;
    if (iterations == 0) { cudaMemcpyAsync(out, color, (size_t)npix * sizeof(float4), cudaMemcpyDeviceToDevice, st); return; }
    const int grid = streaming_grid(npix);
    float4 *iv[2] = { scratch, scratch + npix }, *aux = scratch + 2 * (size_t)npix;
    k_dn_prepare<<<grid, 256, 0, st>>>(W, H, color, albedo_cov, normal_depth, variance, iv[0], aux);
    for (uint32_t k = 0; k < iterations; k++)
        k_dn_atrous<<<grid, 256, 0, st>>>(W, H, 1u << k, iv[k & 1u], normal_depth, aux, sigma_l, sigma_n, sigma_z, iv[(k & 1u) ^ 1u]);
    k_dn_remodulate<<<grid, 256, 0, st>>>(npix, iv[iterations & 1u], albedo_cov, color, out);
}

} // namespace b200pt
