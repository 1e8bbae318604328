// shading.cuh -- device-side restatement of the reference's Slang shading code for sm_90a.
// Every function names the reference lines it implements (SH = PathTracer/Shaders).
// Arithmetic is fp32; operation order follows the Slang source so the GPU and the CPU oracle agree to
// rounding (the only differences are FMA contraction and CUDA-vs-glibc libm ulps).
#pragma once
#include "device_types.h"
#include <math_constants.h>

namespace b200pt {

// SH/Defines.slang:1-17
#define PT_PI         3.1415926535897F
#define PT_1_OVER_PI  0.3183098861837F
#define PT_MAX_DEPTH  1000000u

// ---------------------------------------------------------------- float3 helpers
__device__ __forceinline__ float3 f3(float x, float y, float z) { return make_float3(x, y, z); }
__device__ __forceinline__ float3 f3(float s) { return make_float3(s, s, s); }
__device__ __forceinline__ float3 f3(float4 v) { return make_float3(v.x, v.y, v.z); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 operator*(float3 a, float3 b) { return f3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float3 operator/(float3 a, float3 b) { return f3(a.x / b.x, a.y / b.y, a.z / b.z); }
__device__ __forceinline__ float3 operator*(float3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
#ifdef B200PT_PRECISE
__device__ __forceinline__ float3 operator/(float3 a, float s) { return f3(a.x / s, a.y / s, a.z / s); }
#else   // one reciprocal instead of three divisions (2-ulp class, see Makefile PRECISE)
__device__ __forceinline__ float3 operator/(float3 a, float s) { const float r = 1.0f / s; return f3(a.x * r, a.y * r, a.z * r); }
#endif
__device__ __forceinline__ float3 operator-(float3 a) { return f3(-a.x, -a.y, -a.z); }
__device__ __forceinline__ float dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 cross(float3 a, float3 b) { return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float length(float3 a) { return sqrtf(dot(a, a)); }
#ifdef B200PT_PRECISE
__device__ __forceinline__ float3 normalize(float3 a) { float inv = 1.0f / sqrtf(dot(a, a)); return a * inv; }
#else
__device__ __forceinline__ float3 normalize(float3 a) { float inv = rsqrtf(dot(a, a)); return a * inv; }
#endif
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ float mixf(float x, float y, float a) { return x * (1.0f - a) + y * a; }            // FMix
__device__ __forceinline__ float3 mix3(float3 x, float3 y, float a) { return f3(mixf(x.x, y.x, a), mixf(x.y, y.y, a), mixf(x.z, y.z, a)); }
__device__ __forceinline__ float3 reflect3(float3 i, float3 n) { float d = dot(n, i); return i - n * (2.0f * d); }
__device__ __forceinline__ float3 refract3(float3 i, float3 n, float eta) {
    float d = dot(n, i);
    float k = 1.0f - eta * eta * (1.0f - d * d);
    if (k < 0.0f) return f3(0.0f);
    return i * eta - n * (eta * d + sqrtf(k));
}
// SH/RTCommon.slang:37-45
// cos/sin of the sky angles are evaluated once on the host (engine.cu) instead of per call.
__device__ __forceinline__ float3 rotate3_cs(float3 v, float3 axis, float c, float s) {
    float3 n = normalize(axis);
    return (v * c + cross(n, v) * s) + (n * dot(n, v)) * (1.0f - c);
}
// libm calls with large inlined slow paths are funnelled through single out-of-line copies: k_shade's code must stay
// within the instruction caches (ncu round 1: 189 KB of SASS, stall_no_instruction 20 warps/issue).
static __device__ __noinline__ float2 pt_sincos2(float x) { float s, c; sincosf(x, &s, &c); return make_float2(s, c); }   // by value: no stack round trip
__device__ __forceinline__ void pt_sincos(float x, float *s, float *c) { const float2 r = pt_sincos2(x); *s = r.x; *c = r.y; }
static __device__ __noinline__ float pt_pow(float x, float y) { return powf(x, y); }

// ---------------------------------------------------------------- RNG  SH/Sampler.slang:4-9,21-43
__device__ __forceinline__ uint32_t pcg_hash(uint32_t seed) {
    uint32_t state = seed * 747796405u + 2891336453u;
    uint32_t word = ((state >> ((state >> 28u) + 4u)) ^ state) * 277803737u;
    return (word >> 22u) ^ word;
}
struct Rng {
    uint32_t s;
    __device__ __forceinline__ float next() { s = pcg_hash(s); return (float)s / 4294967296.0f; }   // float(UINT_MAX) == 2^32 (Q12)
    __device__ __forceinline__ uint32_t next_u32() { s = pcg_hash(s); return s; }                    // Sampler::PCG(), SH/Sampler.slang:23-27
};
// SH/Sampler.slang:115-133
__device__ __forceinline__ float3 random_sphere(Rng &r) {
    float u1 = r.next(), u2 = r.next();
    float theta = 2.0f * PT_PI * u1;
    float z = 1.0f - 2.0f * u2;
    float rad = sqrtf(1.0f - z * z);
    float s, c; pt_sincos(theta, &s, &c);
    return f3(rad * c, rad * s, z);
}
// SH/Sampler.slang:143-166
__device__ __forceinline__ float3 ggx_sample_vndf(Rng &r, float3 Ve, float Ax, float Ay) {
    float u1 = r.next(), u2 = r.next();
    float3 Vh = normalize(f3(Ax * Ve.x, Ay * Ve.y, fabsf(Ve.z)));
    float lensq = Vh.x * Vh.x + Vh.y * Vh.y;
    float3 T1 = lensq > 0.0f ? f3(-Vh.y, Vh.x, 0.0f) * (1.0f / sqrtf(lensq)) : f3(1.0f, 0.0f, 0.0f);
    float3 T2 = cross(Vh, T1);
    float rad = sqrtf(u1);
    float phi = 2.0f * PT_PI * u2;
    float sp, cp; pt_sincos(phi, &sp, &cp);
    float t1 = rad * cp, t2 = rad * sp;
    float s = 0.5f * (1.0f + Vh.z);
    t2 = (1.0f - s) * sqrtf(1.0f - t1 * t1) + s * t2;
    float3 Nh = (T1 * t1 + T2 * t2) + Vh * sqrtf(fmaxf(0.0f, 1.0f - t1 * t1 - t2 * t2));
    return normalize(f3(Ax * Nh.x, Ay * Nh.y, fmaxf(0.0f, Nh.z)));
}
// SH/Sampler.slang:169-193
__device__ __forceinline__ float3 sample_henyey_greenstein(Rng &r, float3 incident, float G) {
    float rx = r.next(), ry = r.next();
    float cosTheta;
    if (fabsf(G) < 1e-5f) cosTheta = 2.0f * rx - 1.0f;
    else { float sq = (1.0f - G * G) / (1.0f - G + 2.0f * G * rx); cosTheta = (1.0f + G * G - sq * sq) / (2.0f * G); }
    float phi = 2.0f * PT_PI * ry;
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    float sp, cp; pt_sincos(phi, &sp, &cp);
    float3 nd = f3(sinTheta * cp, sinTheta * sp, cosTheta);
    float3 up = fabsf(incident.y) < 0.9999999f ? f3(0, 1, 0) : f3(0, 0, 1);
    float3 tangent = normalize(cross(up, incident));
    float3 bitangent = cross(incident, tangent);
    return normalize((tangent * nd.x + bitangent * nd.y) + incident * nd.z);
}

// ---------------------------------------------------------------- software texture units (SURVEY Appendix A)
__device__ __forceinline__ float tex_mix(float p, float q, float w) { return p + w * (q - p); }
__device__ __forceinline__ int wrap_repeat(int i, int n) {
    if ((unsigned)i < (unsigned)n) return i;        // interior texel: skip the integer division (same result)
    int m = i % n; return m < 0 ? m + n : m;
}
__device__ __forceinline__ int clampi(int i, int lo, int hi) { return i < lo ? lo : (i > hi ? hi : i); }

// UNORM8 texel -> float, correctly rounded like the texture unit's conversion and the host's c / 255 of 1x1 textures (DevMaterial::cbase ..):
// under -prec-div=false a plain c / 255.0f is the approximate division, off by an ulp for about half of the 256 values, and the per-hit
// path then differed from the per-material one (k_prepare_materials) on the same texels.  c * (1/255) is off for 126 of the values; one
// FMA residual step rounds all 256 correctly (checked exhaustively), at two FMAs instead of a full division.
__device__ __forceinline__ float unorm8(uint8_t c) {
    const float x = (float)c, r = 0x1.010102p-8f;                           // fp32(1/255)
    const float q = __fmul_rn(x, r);
    return __fmaf_rn(__fmaf_rn(-q, 255.0f, x), r, q);
}
// RGBA8 / R8 UNORM, bilinear, REPEAT (PT/PathTracer.cpp:84-91). R8 -> (r,0,0,1).
static __device__ __noinline__ float4 tex_sample_u8(const DevTexture t, float u, float v) {
    const int W = (int)t.w, H = (int)t.h;
    if (W == 1 && H == 1) {     // 1x1 defaults (PT/PathTracer.cpp:1557-1621): bilinear of equal texels is the texel
        if (t.c == 4) { uchar4 p = *reinterpret_cast<const uchar4 *>(t.data); return make_float4(unorm8(p.x), unorm8(p.y), unorm8(p.z), unorm8(p.w)); }
        return make_float4(unorm8(t.data[0]), 0.0f, 0.0f, 1.0f);
    }
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx = floorf(x), fy = floorf(y);
    float ax = x - fx, ay = y - fy;
    int x0 = wrap_repeat((int)fx, W), x1 = wrap_repeat((int)fx + 1, W);
    int y0 = wrap_repeat((int)fy, H), y1 = wrap_repeat((int)fy + 1, H);
    if (t.c == 4) {
        const uchar4 *d = reinterpret_cast<const uchar4 *>(t.data);
        uchar4 p00 = __ldg(d + (size_t)y0 * W + x0), p10 = __ldg(d + (size_t)y0 * W + x1);
        uchar4 p01 = __ldg(d + (size_t)y1 * W + x0), p11 = __ldg(d + (size_t)y1 * W + x1);
        float4 o;
        o.x = tex_mix(tex_mix(unorm8(p00.x), unorm8(p10.x), ax), tex_mix(unorm8(p01.x), unorm8(p11.x), ax), ay);
        o.y = tex_mix(tex_mix(unorm8(p00.y), unorm8(p10.y), ax), tex_mix(unorm8(p01.y), unorm8(p11.y), ax), ay);
        o.z = tex_mix(tex_mix(unorm8(p00.z), unorm8(p10.z), ax), tex_mix(unorm8(p01.z), unorm8(p11.z), ax), ay);
        o.w = tex_mix(tex_mix(unorm8(p00.w), unorm8(p10.w), ax), tex_mix(unorm8(p01.w), unorm8(p11.w), ax), ay);
        return o;
    }
    const uint8_t *d = t.data;
    float t00 = unorm8(__ldg(d + (size_t)y0 * W + x0)), t10 = unorm8(__ldg(d + (size_t)y0 * W + x1));
    float t01 = unorm8(__ldg(d + (size_t)y1 * W + x0)), t11 = unorm8(__ldg(d + (size_t)y1 * W + x1));
    return make_float4(tex_mix(tex_mix(t00, t10, ax), tex_mix(t01, t11, ax), ay), 0.0f, 0.0f, 1.0f);
}
// RGBA32F env map, bilinear, REPEAT
__device__ __forceinline__ float4 env_sample(const DevScene &sc, float u, float v) {
    const int W = (int)sc.envW, H = (int)sc.envH;
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx = floorf(x), fy = floorf(y);
    float ax = x - fx, ay = y - fy;
    int x0 = wrap_repeat((int)fx, W), x1 = wrap_repeat((int)fx + 1, W);
    int y0 = wrap_repeat((int)fy, H), y1 = wrap_repeat((int)fy + 1, H);
    float4 p00 = __ldg(sc.env + (size_t)y0 * W + x0), p10 = __ldg(sc.env + (size_t)y0 * W + x1);
    float4 p01 = __ldg(sc.env + (size_t)y1 * W + x0), p11 = __ldg(sc.env + (size_t)y1 * W + x1);
    float4 o;
    o.x = tex_mix(tex_mix(p00.x, p10.x, ax), tex_mix(p01.x, p11.x, ax), ay);
    o.y = tex_mix(tex_mix(p00.y, p10.y, ax), tex_mix(p01.y, p11.y, ax), ay);
    o.z = tex_mix(tex_mix(p00.z, p10.z, ax), tex_mix(p01.z, p11.z, ax), ay);
    o.w = tex_mix(tex_mix(p00.w, p10.w, ax), tex_mix(p01.w, p11.w, ax), ay);
    return o;
}
// R32F 2D array, linear CLAMP_TO_EDGE in (x,y), nearest-even layer (PT/PathTracer.cpp:93-94,871-937)
__device__ __forceinline__ float lut_sample(const float *lut, int W, int H, int L, float u, float v, float layer) {
    int li = clampi(__float2int_rn(layer), 0, L - 1);
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx = floorf(x), fy = floorf(y);
    float ax = x - fx, ay = y - fy;
    int x0 = clampi((int)fx, 0, W - 1), x1 = clampi((int)fx + 1, 0, W - 1);
    int y0 = clampi((int)fy, 0, H - 1), y1 = clampi((int)fy + 1, 0, H - 1);
    const float *p = lut + (size_t)li * W * H;
    return tex_mix(tex_mix(__ldg(p + y0 * W + x0), __ldg(p + y0 * W + x1), ax), tex_mix(__ldg(p + y1 * W + x0), __ldg(p + y1 * W + x1), ax), ay);
}

__device__ __forceinline__ float power_heuristic(float a, float b) { return (a * a) / ((a * a) + (b * b)); }   // SH/RTCommon.slang:124-127
// SH/RTCommon.slang:129-136
__device__ __forceinline__ void direction_to_uv(float3 d, float &u, float &v) {
    float gamma = asinf(d.y);
    float theta = atan2f(d.x, -d.z);
    u = theta * PT_1_OVER_PI * 0.5f + 0.5f;
    v = gamma * PT_1_OVER_PI + 0.5f;
}

// ---------------------------------------------------------------- transforms
__device__ __forceinline__ float3 xf_point(const float *m, float3 p) {   // row-major 3x4
    return f3(m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3] * 1.0f,
              m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7] * 1.0f,
              m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11] * 1.0f);
}
__device__ __forceinline__ float3 xf_normal(const float *w, float3 n) {  // mul(n, WorldToObject()).xyz
    return f3(n.x * w[0] + n.y * w[3] + n.z * w[6],
              n.x * w[1] + n.y * w[4] + n.z * w[7],
              n.x * w[2] + n.y * w[5] + n.z * w[8]);
}
__device__ __forceinline__ float3 mat4_point(const float *t, float3 p) { // column-major 4x4, w=1
    return f3(t[0] * p.x + t[4] * p.y + t[8] * p.z + t[12] * 1.0f,
              t[1] * p.x + t[5] * p.y + t[9] * p.z + t[13] * 1.0f,
              t[2] * p.x + t[6] * p.y + t[10] * p.z + t[14] * 1.0f);
}
__device__ __forceinline__ float3 mat4_dir(const float *t, float3 p) {   // w=0
    return f3(t[0] * p.x + t[4] * p.y + t[8] * p.z + t[12] * 0.0f,
              t[1] * p.x + t[5] * p.y + t[9] * p.z + t[13] * 0.0f,
              t[2] * p.x + t[6] * p.y + t[10] * p.z + t[14] * 0.0f);
}

// ---------------------------------------------------------------- Surface  SH/Surface.slang:6-159
struct Surface {
    float3 WorldPos; float u, v;
    float3 Normal, Tangent, Bitangent, GeometryNormal;
    float3 P1, P2, P3;
    bool HitFromInside;
    __device__ __forceinline__ float3 tangent_to_world(float3 a) const { return normalize((Tangent * a.x + Bitangent * a.y) + Normal * a.z); }
    __device__ __forceinline__ float3 world_to_tangent(float3 a) const { return normalize(f3(dot(a, Tangent), dot(a, Bitangent), dot(a, Normal))); }
};

__device__ __forceinline__ b200pt_vertex load_vertex(const b200pt_vertex *p) {
    const float4 *q = reinterpret_cast<const float4 *>(p);
    float4 a = __ldg(q), b = __ldg(q + 1);
    b200pt_vertex v;
    v.Position[0] = a.x; v.Position[1] = a.y; v.Position[2] = a.z; v.Normal[0] = a.w;
    v.Normal[1] = b.x; v.Normal[2] = b.y; v.TexCoord[0] = b.z; v.TexCoord[1] = b.w;
    return v;
}

__device__ __forceinline__ void surface_init(Surface &sf, const DevScene &sc, const DevConfig &cfg, const DevInstance &in, const float4 (&g)[7],
                                             float bu, float bv, float3 rayDir, const DevMaterial &dm) {
    // g = ShadeTri of the hit triangle (object-space vertices, SH/Surface.slang:33-41)
    b200pt_vertex A, B, C;
    A.Position[0] = g[0].x; A.Position[1] = g[0].y; A.Position[2] = g[0].z; B.Position[0] = g[1].x; B.Position[1] = g[1].y; B.Position[2] = g[1].z;
    C.Position[0] = g[2].x; C.Position[1] = g[2].y; C.Position[2] = g[2].z;
    A.Normal[0] = g[3].x; A.Normal[1] = g[3].y; A.Normal[2] = g[3].z; B.Normal[0] = g[4].x; B.Normal[1] = g[4].y; B.Normal[2] = g[4].z;
    C.Normal[0] = g[5].x; C.Normal[1] = g[5].y; C.Normal[2] = g[5].z;
    A.TexCoord[0] = g[3].w; A.TexCoord[1] = g[4].w; B.TexCoord[0] = g[5].w; B.TexCoord[1] = g[6].x; C.TexCoord[0] = g[6].y; C.TexCoord[1] = g[6].z;
    float b0 = 1.0f - bu - bv, b1 = bu, b2 = bv;                                  // SH/ClosestHit.slang:45
    float3 p1 = f3(A.Position[0], A.Position[1], A.Position[2]), p2 = f3(B.Position[0], B.Position[1], B.Position[2]), p3 = f3(C.Position[0], C.Position[1], C.Position[2]);
    sf.P1 = p1; sf.P2 = p2; sf.P3 = p3;
    float3 lp = (p1 * b0 + p2 * b1) + p3 * b2;                                    // :43
    sf.WorldPos = xf_point(in.o2w, lp);                                           // :44
    sf.u = A.TexCoord[0] * b0 + B.TexCoord[0] * b1 + C.TexCoord[0] * b2;          // :46
    sf.v = A.TexCoord[1] * b0 + B.TexCoord[1] * b1 + C.TexCoord[1] * b2;
    float3 gn = normalize(cross(p2 - p1, p3 - p1));                               // :48
    gn = normalize(xf_normal(in.w2o, gn));                                        // :49
    float3 n;
    if (cfg.UseOnlyGeometryNormals) n = gn;                                       // :53
    else {
        float3 n1 = f3(A.Normal[0], A.Normal[1], A.Normal[2]), n2 = f3(B.Normal[0], B.Normal[1], B.Normal[2]), n3 = f3(C.Normal[0], C.Normal[1], C.Normal[2]);
        n = normalize((n1 * b0 + n2 * b1) + n3 * b2);                             // :59
        n = normalize(xf_normal(in.w2o, n));                                      // :60
    }
    float3 view = -rayDir;                                                        // :64
    if (dot(gn, view) < 0.0f) { n = -n; gn = -gn; sf.HitFromInside = true; } else sf.HitFromInside = false;   // :66-76
    float3 up = fabsf(n.z) < 0.9999999f ? f3(0, 0, 1) : f3(1, 0, 0);             // :78
    sf.GeometryNormal = gn; sf.Normal = n;
    sf.Tangent = normalize(cross(up, n));                                         // :82
    sf.Bitangent = normalize(cross(n, sf.Tangent));                               // :83
    if (!cfg.UseOnlyGeometryNormals) {                                            // :85-90 (Q10)
        const float4 t = (dm.const_mask & 2u) ? dm.cnormal : tex_sample_u8(sc.textures[dm.m.NormalTextureIndex], sf.u, sf.v);
        sf.Normal = sf.tangent_to_world(f3(t.x * 2.0f - 1.0f, t.y * 2.0f - 1.0f, t.z * 2.0f - 1.0f));
    }
    if (dot(sf.Normal, view) < 0.0f) {                                            // :92-100
        sf.Normal = normalize(sf.Normal - view * (dot(sf.Normal, view) - 0.01f));
    }
    float3 perfect = normalize(reflect3(-view, sf.Normal));                       // :102
    if (dot(perfect, gn) < 0.0f) {                                                // :103-112
        float dp = dot(sf.Normal, gn);
        sf.Normal = normalize(sf.Normal + gn * (0.1f + dp));
    }
    sf.Tangent = normalize(cross(sf.Normal, up));                                 // :115
    sf.Bitangent = normalize(cross(sf.Normal, sf.Tangent));                       // :116
}
// SH/Surface.slang:140-147
__device__ __forceinline__ void surface_rotate_tangents(Surface &sf, float deg) {
    float rot = deg * (PT_PI / 180.0f);
    if (deg == 0.0f) { sf.Bitangent = cross(sf.Tangent, sf.Normal); return; }   // cos 0 = 1, sin 0 = 0: T*1 + x*0 + y*0 == T exactly
    float s, c; pt_sincos(rot, &s, &c);
    float3 T = sf.Tangent, N = sf.Normal;
    float3 r = (T * c + cross(N, T) * s) + (N * dot(N, T)) * (1.0f - c);
    sf.Tangent = r;
    sf.Bitangent = cross(r, N);
}

// ---------------------------------------------------------------- Material  SH/Material.slang
struct Mat {
    float3 BaseColor, EmissiveColor, SpecularColor;
    float Metallic, Roughness, IOR, Transmission, Anisotropy, AnisotropyRotation;
    float Eta, Ax, Ay;
    float pm, pd, pg;        // lobe probabilities (SH/Material.slang:169-177); uv-independent for constant textures, so they live here
};
struct Eval { float3 BxDF; float PDF; };
struct BSample { float3 L; float3 BxDF; float PDF; };

// The part of Material construction that needs texels (SH/Material.slang:39-77) + the lobe probabilities (:169-177).  One function,
// used per hit for textured materials and once per material (k_prepare_materials) for constant ones: identical arithmetic either way.
__device__ __forceinline__ void material_apply_texels(Mat &m, float4 tb, float rough_t, float metal_t, float4 te) {
    m.IOR = fmaxf(m.IOR, 1.000001f);
    m.BaseColor = m.BaseColor * f3(pt_pow(tb.x, 2.2f), pt_pow(tb.y, 2.2f), pt_pow(tb.z, 2.2f));
    m.Roughness *= rough_t;                                                       // Q8, Q9
    m.Metallic *= metal_t;
    m.EmissiveColor = m.EmissiveColor * f3(te.x, te.y, te.z);
    float aspect = sqrtf(1.0f - sqrtf(m.Anisotropy) * 0.9f);
    m.Ax = fmaxf(0.00001f, m.Roughness / aspect);
    m.Ay = fmaxf(0.00001f, m.Roughness * aspect);
    m.pm = m.Metallic;
    m.pd = (1.0f - m.Metallic) * (1.0f - m.Transmission);
    m.pg = (1.0f - m.Metallic) * m.Transmission;
    const float sum = m.pm + m.pd + m.pg;
    m.pm /= sum; m.pd /= sum; m.pg /= sum;
}
__device__ __forceinline__ void material_load_constants(Mat &m, const b200pt_material &src) {
    m.BaseColor = f3(src.BaseColor[0], src.BaseColor[1], src.BaseColor[2]);
    m.EmissiveColor = f3(src.EmissiveColor[0], src.EmissiveColor[1], src.EmissiveColor[2]);
    m.Metallic = src.Metallic; m.Roughness = src.Roughness; m.IOR = src.IOR; m.Transmission = src.Transmission;
    m.Anisotropy = src.Anisotropy;
}
// :39-87
__device__ __forceinline__ void material_init(Mat &m, const DevScene &sc, const DevConfig &cfg, const DevMaterial &dm, const Surface &sf) {
    const b200pt_material &src = dm.m;
    m.SpecularColor = f3(src.SpecularColor[0], src.SpecularColor[1], src.SpecularColor[2]);
    m.AnisotropyRotation = src.AnisotropyRotation;
    if (dm.const_mask & 32u) {                                                   // every texture of the material is 1x1: use the per-material results
        const float4 p0 = dm.pre0, p1 = dm.pre1, p2 = dm.pre2, p3 = dm.pre3;
        m.BaseColor = f3(p0); m.Roughness = p0.w; m.EmissiveColor = f3(p1); m.Metallic = p1.w;
        m.Ax = p2.x; m.Ay = p2.y; m.IOR = p2.z; m.pm = p3.x; m.pd = p3.y; m.pg = p3.z;
        m.Transmission = src.Transmission; m.Anisotropy = src.Anisotropy;
    } else {
        material_load_constants(m, src);
        const float4 tb = (dm.const_mask & 1u) ? dm.cbase : tex_sample_u8(sc.textures[src.BaseColorTextureIndex], sf.u, sf.v);
        const float tr = (dm.const_mask & 4u) ? dm.crough : tex_sample_u8(sc.textures[src.RoughnessTextureIndex], sf.u, sf.v).x;
        const float tm = (dm.const_mask & 8u) ? dm.cmetal : tex_sample_u8(sc.textures[src.MetallicTextureIndex], sf.u, sf.v).x;
        const float4 te = (dm.const_mask & 16u) ? dm.cemis : tex_sample_u8(sc.textures[src.EmissiveTextureIndex], sf.u, sf.v);
        material_apply_texels(m, tb, tr, tm, te);
    }
    m.Eta = sf.HitFromInside ? m.IOR : 1.0f / m.IOR;
    if (cfg.FurnaceTestMode) { m.BaseColor = f3(1.0f); m.EmissiveColor = f3(0.0f); m.SpecularColor = f3(1.0f); }   // :78-86 (MediumColor: k_shade_hit)
}
__device__ __forceinline__ float schlick_fresnel(float VdotH) { float m = clampf(1.0f - VdotH, 0.0f, 1.0f); float m2 = m * m; return m2 * m2 * m; }   // :427-432
// :434-449
__device__ __forceinline__ float dielectric_fresnel(float cosI, float eta) {
    float sinT2 = eta * eta * (1.0f - cosI * cosI);
    if (sinT2 > 1.0f) return 1.0f;
    float cosT = sqrtf(fmaxf(1.0f - sinT2, 0.0f));
    float rs = (eta * cosT - cosI) / (eta * cosT + cosI);
    float rp = (eta * cosI - cosT) / (eta * cosI + cosT);
    return 0.5f * (rs * rs + rp * rp);
}
// Per-hit quantities of EvaluateBSDF that do not depend on L.  The shader evaluates the BSDF up to three times per hit
// (sampled direction, sky NEE, light NEE); these values are identical in all three, so they are computed once.  Every
// expression keeps the operand order of the Slang source, so hoisting does not change a single bit.
struct BsdfCtx {
    float pm, pd, pg;          // :169-177 lobe probabilities
    float ax2, ay2, dnorm;     // Ax^2, Ay^2, PI*Ax*Ay            (:394-404)
    float GV;                  // GGXSmithAnisotropic(V)          (:420-423)
    float reflEC, glassEC;     // energy-compensation LUT values  (:203-217, :299-303, :316-320)
    float3 metalEC;            // 1 + BaseColor * (1-E)/E         (:303-304)
    float3 diffuse;            // M_1_OVER_PI * BaseColor         (:284)
    float fourVz;              // 4 * V.z
};
__device__ __forceinline__ float ggx_g1(const Mat &m, float3 V) {                  // :406-423
    float Vz2 = fabsf(V.z) * fabsf(V.z);
    float ax2 = m.Ax * m.Ax, ay2 = m.Ay * m.Ay;
    float nom = -1.0f + sqrtf(1.0f + (ax2 * (V.x * V.x) + ay2 * (V.y * V.y)) / Vz2);
    return 1.0f / (1.0f + nom / 2.0f);
}
__device__ __forceinline__ float ggx_d(const BsdfCtx &c, float3 H) {               // :394-404
    float e = (H.x * H.x) / c.ax2 + (H.y * H.y) / c.ay2 + H.z * H.z;
    return 1.0f / (c.dnorm * (e * e));
}
// Lobe sets (template parameter LOBES of the functions below): a material class (device_types.h: MaterialClass) whose lobe probability is
// exactly 0 contributes exact zeros through `b * p` and `pdf * p` for every finite b, so that lobe's code is dropped from the class's kernel.
constexpr uint32_t LB_M = 1u, LB_D = 2u, LB_G = 4u, LB_ALL = 7u;
__host__ __device__ constexpr uint32_t class_lobes(uint32_t mc) { return mc == MC_DIFFUSE ? LB_D : (mc == MC_METAL ? LB_M : (mc == MC_GLASS ? LB_G : LB_ALL)); }
template <uint32_t LOBES = LB_ALL>
__device__ __forceinline__ void bsdf_ctx_init(BsdfCtx &c, const Mat &m, const DevScene &sc, const DevConfig &cfg, float3 V) {
    c.pm = m.pm; c.pd = m.pd; c.pg = m.pg;                                   // :169-177 (material_apply_texels)
    c.ax2 = m.Ax * m.Ax; c.ay2 = m.Ay * m.Ay; c.dnorm = PT_PI * m.Ax * m.Ay;
    c.GV = ggx_g1(m, V);
    c.reflEC = 1.0f; c.glassEC = 0.0f; c.metalEC = f3(1.0f);
    if (cfg.UseEnergyCompensation) {
        if (LOBES & LB_G) {
            const bool inside = m.Eta > 1.0f;
            const float layer = (clampf(m.IOR, 1.0001f, 2.0f) - 1.0f) * 32.0f;
            c.glassEC = lut_sample(inside ? sc.lut_refract_in : sc.lut_refract_out, 128, 128, 32, sqrtf(V.z), m.Roughness, layer);
        }
        if (LOBES & (LB_M | LB_D)) {
            c.reflEC = lut_sample(sc.lut_reflect, 64, 64, 32, V.z, m.Roughness, m.Anisotropy * 32.0f);
            const float ec = (1.0f - c.reflEC) / c.reflEC;
            c.metalEC = f3(1.0f) + m.BaseColor * f3(ec);
        }
    }
    c.diffuse = m.BaseColor * PT_1_OVER_PI;
    c.fourVz = 4.0f * V.z;
}
// :167-279 (+ :281-387): EvaluateBSDF(V, L)
template <uint32_t LOBES = LB_ALL>
__device__ __forceinline__ Eval eval_bsdf(const Mat &m, const BsdfCtx &c, const DevConfig &cfg, float3 V, float3 L) {
    const bool refracted = L.z < 0.0f;
    Eval out; out.BxDF = f3(0.0f); out.PDF = 0.0f;
    if (!refracted) {
        const float3 H = normalize(V + L);
        const float VdotH = dot(V, H);
        float F = 0.0f;
        if (LOBES & (LB_D | LB_G)) F = dielectric_fresnel(fabsf(VdotH), m.Eta);   // :202
        // EvaluateReflection (:331-351) shared by the metallic, dielectric-specular and glass-reflect lobes
        float rpdf = 0.0f; bool refl = false; float D = 0.0f, GL = 0.0f;
        if (!(L.z <= 1e-5f)) {
            refl = true;
            D = ggx_d(c, H); GL = ggx_g1(m, L);
            rpdf = (c.GV * fmaxf(VdotH, 0.0f) * D / V.z) / (4.0f * VdotH);
        }
        if (LOBES & LB_M) {   // metallic :291-308
            float3 b = f3(0.0f);
            if (refl) {
                const float3 Fm = mix3(m.BaseColor, m.SpecularColor, schlick_fresnel(VdotH));
                b = (((Fm * D) * c.GV) * GL) / c.fourVz;
            }
            if (cfg.UseEnergyCompensation) b = c.metalEC * b;
            out.BxDF = out.BxDF + b * c.pm; out.PDF += rpdf * c.pm;
        }
        if (LOBES & LB_D) {   // diffuse :281-289
            float pdf = L.z * PT_1_OVER_PI;
            const float3 brdf = c.diffuse * L.z;
            pdf *= (L.z > 0.0f) ? 1.0f : 0.0f;
            out.BxDF = out.BxDF + (brdf * c.pd) * (1.0f - F); out.PDF += pdf * c.pd * (1.0f - F);
        }
        float3 spec = f3(0.0f);
        if ((LOBES & (LB_D | LB_G)) && refl) spec = (((m.SpecularColor * D) * c.GV) * GL) / c.fourVz;
        if (LOBES & LB_D) {   // dielectric specular :310-323
            float3 b = spec;
            if (cfg.UseEnergyCompensation) b = b / c.reflEC;
            out.BxDF = out.BxDF + (b * c.pd) * F; out.PDF += rpdf * c.pd * F;
        }
        if (LOBES & LB_G) {   // glass reflect :237-251
            float3 b = spec;
            if (cfg.UseEnergyCompensation && c.glassEC > 0.01f) b = b / c.glassEC;
            out.BxDF = out.BxDF + (b * c.pg) * F; out.PDF += rpdf * c.pg * F;
        }
    } else if (LOBES & LB_G) {   // pg == 0 (no glass lobe): every term below is multiplied by an exact 0
        float3 H = normalize(V * m.Eta + L);
        if (H.z < 0.0f) H = -H;
        const float VdotH = dot(V, H), LdotH = dot(L, H);
        const bool validRefraction = (VdotH > 0.0f && LdotH < 0.0f) || (VdotH < 0.0f && LdotH > 0.0f);   // :185-186
        const float F = dielectric_fresnel(fabsf(VdotH), m.Eta);
        if (validRefraction) {   // glass refract :253-267 + EvaluateRefraction :359-387
            float3 b = f3(0.0f); float pdf = 0.0f;
            if (!(L.z >= 1e-5f)) {
                const float D = ggx_d(c, H);
                const float GL = ggx_g1(m, L);
                const float G = c.GV * GL;
                const float den = LdotH + m.Eta * VdotH;
                const float den2 = den * den;
                const float eta2 = m.Eta * m.Eta;
                const float jac = (eta2 * fabsf(LdotH)) / den2;
                pdf = (c.GV * fabsf(VdotH) * D / V.z) * jac;
                const float k = fabsf(VdotH) * fabsf(LdotH) / fabsf(V.z);
                b = ((((m.BaseColor * D) * G) * eta2) / den2) * k;
            }
            if (cfg.UseEnergyCompensation && c.glassEC > 0.01f) b = b / c.glassEC;
            out.BxDF = out.BxDF + (b * c.pg) * (1.0f - F); out.PDF += pdf * c.pg * (1.0f - F);
        }
    }
    return out;
}
// :94-165
// Direction part of SampleBSDF (:94-160).  Returns false for the "invalid reflection/refraction direction" early-outs
// (:152-160); the BxDF/PDF of a valid direction come from EvaluateBSDF(V, L) (:163), evaluated by the caller.
// LOBES: with pm == 0 the test x1 < pm never holds (x1 >= 0); with pd == 0 the test x1 < pm + pd repeats x1 < pm.  The glass branch stays
// in every class: x1 can be exactly 1.0 (Q12), which falls through to it even when pg == 0.
template <uint32_t LOBES = LB_ALL>
__device__ __forceinline__ bool sample_bsdf_direction(const Mat &m, const BsdfCtx &c, Rng &rng, float3 V, float3 H, float3 &Lout) {
    const float pm = c.pm, pd = c.pd;
    float F = dielectric_fresnel(dot(V, H), m.Eta);
    float x1 = rng.next();
    float3 L; bool refracted = false;
    if ((LOBES & LB_M) && x1 < pm) L = normalize(reflect3(-V, H));
    else if ((LOBES & LB_D) && x1 < pm + pd) {
        if (rng.next() < F) L = normalize(reflect3(-V, H));
        else L = normalize(random_sphere(rng) + f3(0.0f, 0.0f, 1.0f));
    } else {
        if (rng.next() < F) L = normalize(reflect3(-V, H));
        else { L = normalize(refract3(-V, H, m.Eta)); refracted = true; }
    }
    Lout = L;
    if (L.z < 0.0f && !refracted) return false;
    else if (refracted && L.z >= 0.0f) return false;
    return true;
}

// ---------------------------------------------------------------- NEE samplers
// SH/Sampler.slang:287-346, split in two so the dependent DRAM access (random 8-B alias entry out of a 64 MiB table)
// can be issued at the top of the shading kernel and overlap the surface / material set-up.
struct EnvPick { float xy, xz; uint32_t idx; uint2 entry; };
__device__ __forceinline__ void sample_env_begin(const DevScene &sc, Rng &rng, EnvPick &p) {
    const float xx = rng.next(); p.xy = rng.next(); p.xz = rng.next();     // UniformFloat3 (:290)
    const uint32_t size = sc.envW * sc.envH;
    p.idx = min((uint32_t)(xx * (float)size), size - 1u);                   // :297
    p.entry = __ldg(sc.alias + p.idx);                                      // :300
}
__device__ __forceinline__ void sample_env_finish(const DevScene &sc, const DevConfig &cfg, const EnvPick &p, float3 &toLight, float4 &val) {
    float xy = p.xy; const float xz = p.xz;
    const uint32_t width = sc.envW, height = sc.envH;
    const float imp = __uint_as_float(p.entry.y);
    uint32_t envIdx;
    if (xy < imp) { envIdx = p.idx; xy /= imp; }
    else { envIdx = p.entry.x; xy = (xy - imp) / (1.0f - imp); }
    uint32_t px = envIdx % width, py = envIdx / width;
    float u = ((float)px + xy) / (float)width;
    float phi = u * (2.0f * PT_PI) - PT_PI;
    float sinPhi, cosPhi; pt_sincos(phi, &sinPhi, &cosPhi);
    const float2 rc = __ldg(sc.env_row_cos + py);                          // cos(theta0), cos(theta0 + stepTheta): 2 table reads instead of 2 cosf
    float cosTheta = rc.x * (1.0f - xz) + rc.y * xz;
    float theta = acosf(cosTheta);
    float sinTheta = sinf(theta);
    float v = theta * PT_1_OVER_PI;
    float3 d = f3(sinPhi * sinTheta, -cosTheta, -cosPhi * sinTheta);
    d = rotate3_cs(d, f3(0, 1, 0), cfg.cosAz, cfg.sinAz);
    d = rotate3_cs(d, f3(1, 0, 0), cfg.cosAl, cfg.sinAl);
    toLight = d;
    val = env_sample(sc, u, v);
    val.x *= cfg.EnvironmentIntensity; val.y *= cfg.EnvironmentIntensity; val.z *= cfg.EnvironmentIntensity;
}
// SH/Sampler.slang:349-422
// gid: global id of the sampled triangle -- the light ray contributes iff that triangle is the closest hit (SH/ClosestHit.slang:171-176)
__device__ __forceinline__ void sample_emissive(const DevScene &sc, Rng &rng, float3 pos, float3 &toLight, float4 &colorPDF, uint32_t &gid) {
    gid = 0xFFFFFFFFu;
    const uint32_t count = sc.n_emissive;
    if (count == 0) { toLight = f3(0.0f); colorPDF = make_float4(0, 0, 0, 0); return; }
    uint32_t mi = min((uint32_t)floorf(rng.next() * (float)count), count - 1u);
    const DevEmissive &em = sc.emissive[mi];
    const uint32_t tc = em.tri_count;
    uint32_t ti = min((uint32_t)floorf(rng.next() * (float)tc), tc - 1u);
    const float4 *et = reinterpret_cast<const float4 *>(sc.em_tris + (__ldg(sc.em_tri_base + mi) + ti));
    const float4 e0 = __ldg(et), e1 = __ldg(et + 1), e2 = __ldg(et + 2), e3 = __ldg(et + 3);
    gid = __float_as_uint(e3.w);
    const float3 p0 = f3(e0), p1 = f3(e1), p2 = f3(e2);                   // world-space corners (:389-391, transformed once on the host)
    b200pt_vertex A, B, C;
    A.TexCoord[0] = e0.w; A.TexCoord[1] = e1.w; B.TexCoord[0] = e2.w; B.TexCoord[1] = e3.x; C.TexCoord[0] = e3.y; C.TexCoord[1] = e3.z;
    float x0 = rng.next(), x1 = rng.next();
    float su1 = sqrtf(x0);
    float b0 = 1.0f - su1, b1 = x1 * su1, b2 = 1.0f - b0 - b1;
    float3 tp = (p0 * b0 + p1 * b1) + p2 * b2;
    float uu = b0 * A.TexCoord[0] + b1 * B.TexCoord[0] + b2 * C.TexCoord[0];
    float vv = b0 * A.TexCoord[1] + b1 * B.TexCoord[1] + b2 * C.TexCoord[1];
    float3 dl = tp - pos;
    toLight = normalize(dl);
    float3 normal = normalize(cross(p2 - p0, p1 - p0));
    float area = length(cross(p1 - p0, p2 - p0)) * 0.5f;
    float d2 = dot(dl, dl);
    float cosTheta = fabsf(dot(normal, toLight));
    const DevMaterial &dmat = sc.materials[em.material];
    const b200pt_material &mat = dmat.m;
    const float4 te = (dmat.const_mask & 16u) ? dmat.cemis : tex_sample_u8(sc.textures[mat.EmissiveTextureIndex], uu, vv);
    colorPDF.w = d2 / ((float)count * (float)tc * area * cosTheta);
    colorPDF.x = mat.EmissiveColor[0] * te.x; colorPDF.y = mat.EmissiveColor[1] * te.y; colorPDF.z = mat.EmissiveColor[2] * te.z;
}

// ---------------------------------------------------------------- MIS terms (k_shade_hit, k_shade_miss and the test hooks call these)
// Emission of a hit (SH/ClosestHit.slang:265-317) at Depth `depth`, reached from payOrigin with BSDF pdf payPDF: the emissive colour,
// MIS-weighted at Depth > 0 against the light sampler's pdf of the same point, taken with the SHADING normal and floored by the bias.
__device__ __forceinline__ float3 hit_emission(const DevScene &sc, const DevConfig &cfg, const DevInstance &in, const Surface &sf, const Mat &m, bool isLight,
                                               uint32_t depth, float3 payOrigin, float payPDF) {
    float3 e0 = f3(0.0f);
    if (cfg.EnableMeshMIS) {
        if (depth == 0 && isLight) e0 = e0 + m.EmissiveColor;
        else if (isLight) {
            const float3 w1 = xf_point(in.o2w, sf.P1), w2 = xf_point(in.o2w, sf.P2), w3 = xf_point(in.o2w, sf.P3);
            const float area = length(cross(w2 - w1, w3 - w1)) * 0.5f;
            const float3 dl = sf.WorldPos - payOrigin;
            const float d2 = dot(dl, dl);
            const float cosTheta = fabsf(dot(sf.Normal, normalize(payOrigin - sf.WorldPos)));
            float lp = (1.0f / (float)sc.n_emissive) * (1.0f / (float)in.emissive_tri_count) * (1.0f / area) * (d2 / cosTheta);
            lp = fmaxf(lp, cfg.EmissiveMeshSamplingPDFBias);
            e0 = e0 + m.EmissiveColor * power_heuristic(payPDF, lp);
        }
    } else e0 = e0 + m.EmissiveColor;
    return e0;
}
// One NEE term (SH/ClosestHit.slang:341-344, :366-369): BxDF * radiance / pdf, MIS-weighted against the BSDF pdf of the same direction
__device__ __forceinline__ float3 nee_term(const Eval &e, float4 lv) { return (((e.BxDF * 1.0f) * f3(lv)) / lv.w) * power_heuristic(lv.w, e.PDF); }
// What a path whose segment missed receives (SH/Miss.slang:8-76): the environment seen along dir (inverse sky rotation, then the
// lat-long lookup), times the intensity, MIS-weighted at Depth > 0 against the sky sampler's pdf (.w of the lookup, returned in .w)
__device__ __forceinline__ float4 miss_emission(const DevScene &sc, const DevConfig &cfg, float3 dir, uint32_t depth, float payPDF) {
    float4 c;
    if (cfg.EnableAtmosphere) c = make_float4(0, 0, 0, 1);                  // SH/Miss.slang:11-14: with the atmosphere a miss emits nothing
    else if (cfg.ShowEnvMapDirectly || depth > 0) {
        float3 r = rotate3_cs(dir, f3(1, 0, 0), cfg.cosAl, -cfg.sinAl);    // Rotate(dir, X, -altitude): cos is even, sin odd
        r = rotate3_cs(r, f3(0, 1, 0), cfg.cosAz, -cfg.sinAz);
        float u, v; direction_to_uv(r, u, v);
        c = env_sample(sc, u, v);
    } else c = make_float4(0, 0, 0, 1);
    float3 em = f3(c.x * cfg.EnvironmentIntensity, c.y * cfg.EnvironmentIntensity, c.z * cfg.EnvironmentIntensity);
    if (cfg.FurnaceTestMode && !cfg.EnableAtmosphere) em = f3(1.0f);
    if (cfg.EnableSkyMIS && depth > 0 && !cfg.EnableAtmosphere) em = em * power_heuristic(payPDF, c.w);
    return make_float4(em.x, em.y, em.z, c.w);
}

} // namespace b200pt
