// shade_query.cu -- shading test hooks: b200pt_shade_query runs caller-given hits through one shading step of k_shade_hit, b200pt_miss_query
// caller-given directions through k_shade_miss's miss shading.
// Every step calls the __device__ functions the renderer's kernels call (surface_init, material_init, surface_rotate_tangents, bsdf_ctx_init,
// sample_env_begin / _finish, sample_emissive, ggx_sample_vndf, sample_bsdf_direction, eval_bsdf, hit_emission, nee_term, miss_emission), with
// the LOBES argument of the hit triangle's class kernel, in k_shade_hit's draw order.  Only the geometry-normal rejection, a comparison k_shade_hit
// writes inline, is repeated here.
#include "shading.cuh"
#include "kernels.h"
#include <algorithm>

namespace b200pt {

namespace {

constexpr int THREADS = 128;

__device__ __forceinline__ void put3(float *o, float3 a) { o[0] = a.x; o[1] = a.y; o[2] = a.z; }
__device__ __forceinline__ void put_eval(float *o, const Eval &e) { put3(o, e.BxDF); o[3] = e.PDF; }

// k_shade_hit's body for one hit at Depth 1 outside any medium (SH/ClosestHit.slang:40-238), without the shadow queries
template <uint32_t LOBES>
__device__ __forceinline__ void shade_one(const DevScene &sc, const DevConfig &cfg, const ShadeQuery &q, uint32_t i, float *o) {
    const uint32_t gid = q.gid[i];
    const float3 rd = normalize(f3(q.dir[3 * i], q.dir[3 * i + 1], q.dir[3 * i + 2]));
    const float3 payOrigin = f3(q.org[3 * i], q.org[3 * i + 1], q.org[3 * i + 2]);
    const float payPDF = q.pay_pdf[i];
    Rng rng; rng.s = q.rng[i];
    EnvPick ep;
    const bool envEarly = cfg.EnableSkyMIS != 0u;                            // no medium, no atmosphere: the sky draws come first
    if (envEarly) sample_env_begin(sc, rng, ep);
    float4 g[7];
    const float4 *gp = reinterpret_cast<const float4 *>(sc.shade_tris + gid);
    #pragma unroll
    for (int k = 0; k < 7; k++) g[k] = gp[k];
    const DevInstance &in = sc.instances[__float_as_uint(g[0].w)];
    const DevMaterial &cm = sc.materials[__float_as_uint(g[2].w)];
    Surface sf;
    surface_init(sf, sc, cfg, in, g, q.uv[2 * i], q.uv[2 * i + 1], rd, cm);
    Mat m;
    material_init(m, sc, cfg, cm, sf);
    const bool isLight = m.EmissiveColor.x > 0.0f || m.EmissiveColor.y > 0.0f || m.EmissiveColor.z > 0.0f;
    surface_rotate_tangents(sf, m.AnisotropyRotation);
    put3(o + B200PT_SQ_N, sf.Normal); put3(o + B200PT_SQ_T, sf.Tangent); put3(o + B200PT_SQ_B, sf.Bitangent); put3(o + B200PT_SQ_NG, sf.GeometryNormal);
    o[B200PT_SQ_INSIDE] = sf.HitFromInside ? 1.0f : 0.0f;
    o[B200PT_SQ_AX] = m.Ax; o[B200PT_SQ_AY] = m.Ay; o[B200PT_SQ_ETA] = m.Eta; o[B200PT_SQ_PM] = m.pm; o[B200PT_SQ_PD] = m.pd; o[B200PT_SQ_PG] = m.pg;
    put3(o + B200PT_SQ_BASECOLOR, m.BaseColor); o[B200PT_SQ_ROUGHNESS] = m.Roughness;

    put3(o + B200PT_SQ_POS, sf.WorldPos);
    const float3 e0 = hit_emission(sc, cfg, in, sf, m, isLight, 1u, payOrigin, payPDF);   // emission :265-317, Depth != 0
    put3(o + B200PT_SQ_EMITTED, e0);

    float3 V = normalize(-rd);
    V = sf.world_to_tangent(V);
    BsdfCtx bc;
    bsdf_ctx_init<LOBES>(bc, m, sc, cfg, V);
    Eval evS; evS.BxDF = f3(0.0f); evS.PDF = 0.0f;
    float3 Ls = f3(0.0f), H = f3(0.0f); bool validDir = false;
    uint32_t lgid = 0xFFFFFFFFu;
    for (int k = 0; k < 3; k++) {                                           // sky draw, light draw, BSDF draw
        float3 toW = f3(0.0f), dk = f3(0.0f); float4 lv = make_float4(0, 0, 0, 0);
        bool need = false;
        if (k == 0) {
            if (cfg.EnableSkyMIS) {
                sample_env_finish(sc, cfg, ep, toW, lv);
                lv.x *= cfg.EnvironmentIntensity; lv.y *= cfg.EnvironmentIntensity; lv.z *= cfg.EnvironmentIntensity;   // Q7
                dk = sf.world_to_tangent(toW);
                need = lv.w > 0.0f;
                put3(o + B200PT_SQ_SKY_L, dk); put3(o + B200PT_SQ_SKY_W, toW);
            }
        } else if (k == 1) {
            if (cfg.EnableMeshMIS && !isLight) {
                sample_emissive(sc, rng, sf.WorldPos, toW, lv, lgid);
                put3(o + B200PT_SQ_LIGHT_W, toW);
                if (lv.w > 0.0f) { dk = sf.world_to_tangent(toW); need = true; put3(o + B200PT_SQ_LIGHT_L, dk); }
            }
        } else {
            H = ggx_sample_vndf(rng, V, m.Ax, m.Ay);
            validDir = sample_bsdf_direction<LOBES>(m, bc, rng, V, H, Ls);
            dk = Ls; need = validDir;
        }
        Eval e; e.BxDF = f3(0.0f); e.PDF = 0.0f;
        if (need) e = eval_bsdf<LOBES>(m, bc, cfg, V, dk);
        if (k == 2) { evS = e; break; }
        const bool contributes = need && e.PDF > 0.0f;
        const float3 c = contributes ? nee_term(e, lv) : f3(0.0f);
        const int base = k == 0 ? B200PT_SQ_SKY_LV : B200PT_SQ_LIGHT_LV;     // LV, EVAL and C follow each other for both draws
        o[base] = lv.x; o[base + 1] = lv.y; o[base + 2] = lv.z; o[base + 3] = lv.w;
        put_eval(o + base + 4, e); put3(o + base + 8, c);
    }
    o[B200PT_SQ_LIGHT_GID] = __uint_as_float(lgid);
    put3(o + B200PT_SQ_V, V); put3(o + B200PT_SQ_H, H);
    const float3 L = validDir ? Ls : f3(0.0f);
    put3(o + B200PT_SQ_BSDF_L, L); put_eval(o + B200PT_SQ_BSDF_EVAL, evS);
    o[B200PT_SQ_VALID] = validDir ? 1.0f : 0.0f;
    const bool wasRefracted = L.z < 0.0f;                                   // :220-238
    const float3 scatterW = sf.tangent_to_world(L);
    const bool rejected = !wasRefracted && dot(scatterW, sf.GeometryNormal) < 0.0f;
    if (rejected) { evS.PDF = 0.0f; evS.BxDF = f3(0.0f); }
    put3(o + B200PT_SQ_SCATTER, scatterW); put_eval(o + B200PT_SQ_SAMPLE, evS);
    o[B200PT_SQ_REFRACTED] = wasRefracted ? 1.0f : 0.0f;
    o[B200PT_SQ_ENTERED] = (wasRefracted && !sf.HitFromInside) ? 1.0f : 0.0f;
    o[B200PT_SQ_REJECTED] = rejected ? 1.0f : 0.0f;
    if (q.L) {
        const float3 t = sf.world_to_tangent(f3(q.L[3 * i], q.L[3 * i + 1], q.L[3 * i + 2]));
        put3(o + B200PT_SQ_USER_L, t); put_eval(o + B200PT_SQ_USER_EVAL, eval_bsdf<LOBES>(m, bc, cfg, V, t));
    }
    o[B200PT_SQ_RNG] = __uint_as_float(rng.s);
}

__global__ void __launch_bounds__(THREADS) k_shade_query(DevScene sc, DevConfig cfg, ShadeQuery q) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += gridDim.x * blockDim.x) {
        float *o = q.out + (size_t)i * B200PT_SQ_STRIDE;
        for (int k = 0; k < B200PT_SQ_STRIDE; k++) o[k] = 0.0f;
        const uint32_t cls = q.force_general ? (uint32_t)MC_GENERAL : (uint32_t)sc.tri_class[q.gid[i]];   // as k_extend's hit code reads it
        o[B200PT_SQ_CLASS] = (float)cls;
        switch (cls) {                                                      // the LOBES of k_shade_hit<CLASS>
        case MC_DIFFUSE: shade_one<class_lobes(MC_DIFFUSE)>(sc, cfg, q, i, o); break;
        case MC_METAL: shade_one<class_lobes(MC_METAL)>(sc, cfg, q, i, o); break;
        case MC_GLASS: shade_one<class_lobes(MC_GLASS)>(sc, cfg, q, i, o); break;
        default: shade_one<class_lobes(MC_GENERAL)>(sc, cfg, q, i, o); break;
        }
    }
}

// k_shade_miss's miss shading (miss_emission) for caller-given directions, depths and BSDF pdfs: emitted RGB and the env pdf
__global__ void __launch_bounds__(THREADS) k_miss_query(DevScene sc, DevConfig cfg, MissQuery q) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < q.n; i += gridDim.x * blockDim.x) {
        const float4 r = miss_emission(sc, cfg, f3(q.dir[3 * i], q.dir[3 * i + 1], q.dir[3 * i + 2]), q.depth[i], q.pay_pdf[i]);
        float *o = q.out + (size_t)i * B200PT_MQ_STRIDE;
        put3(o + B200PT_MQ_RGB, f3(r)); o[B200PT_MQ_PDF] = r.w;
    }
}

} // namespace

int launch_miss_query(const DevScene &sc, const DevConfig &cfg, const MissQuery &q, cudaStream_t st) {
    if (q.n == 0) return 0;
    const int grid = (int)std::min<uint32_t>((q.n + THREADS - 1) / THREADS, 1024u);
    k_miss_query<<<grid, THREADS, 0, st>>>(sc, cfg, q);
    return (int)cudaGetLastError();
}

int launch_shade_query(const DevScene &sc, const DevConfig &cfg, const ShadeQuery &q, cudaStream_t st) {
    if (q.n == 0) return 0;
    const int grid = (int)std::min<uint32_t>((q.n + THREADS - 1) / THREADS, 1024u);
    k_shade_query<<<grid, THREADS, 0, st>>>(sc, cfg, q);
    return (int)cudaGetLastError();
}

} // namespace b200pt
