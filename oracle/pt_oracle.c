/*
 * pt_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE ONLY; see pt_oracle.h for the pin status).
 * Restates, function by function, the reference's Slang integrator.  Every function cites the
 * reference file:line it follows (paths relative to the reference repository; SH = PathTracer/Shaders,
 * PT = PathTracer).  Quirks Q1..Q16 of SURVEY.md Appendix B are kept verbatim.
 */
#include "pt_oracle.h"
#include "orc_math.h"
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <unistd.h>

/* ------------------------------------------------------------------------------------------------
 * RNG: SH/Sampler.slang:4-9, 21-100
 * ---------------------------------------------------------------------------------------------- */
typedef struct { uint32_t seed; } Rng;

uint32_t orc_pcg_hash(uint32_t seed) {
    uint32_t state = seed * 747796405u + 2891336453u;
    uint32_t word = ((state >> ((state >> 28u) + 4u)) ^ state) * 277803737u;
    return (word >> 22u) ^ word;
}
static inline uint32_t rng_pcg(Rng *r) { r->seed = orc_pcg_hash(r->seed); return r->seed; }
/* SH/Sampler.slang:38-43: float(hash) / float(UINT_MAX); float(UINT_MAX) rounds to 2^32 (Q12: result in [0,1]) */
static inline float rng_f(Rng *r) { return (float)rng_pcg(r) / 4294967296.0f; }

void orc_rng_floats(uint32_t seed, uint32_t n, float *out) {
    Rng r = { seed };
    for (uint32_t i = 0; i < n; i++) out[i] = rng_f(&r);
}

/* SH/Sampler.slang:103-112 */
static inline void rng_circle(Rng *r, float *ox, float *oy) {
    float u1 = rng_f(r), u2 = rng_f(r);
    float theta = 2.0f * ORC_PI * u1;
    float rad = sqrtf(u2);
    *ox = rad * cosf(theta); *oy = rad * sinf(theta);
}
/* SH/Sampler.slang:115-133 */
static inline v3 rng_sphere(Rng *r) {
    float u1 = rng_f(r), u2 = rng_f(r);
    float theta = 2.0f * ORC_PI * u1;
    float z = 1.0f - 2.0f * u2;
    float rad = sqrtf(1.0f - z * z);
    return V3(rad * cosf(theta), rad * sinf(theta), z);
}
/* SH/Sampler.slang:143-166 (Heitz 2018 VNDF) */
static inline v3 rng_ggx_vndf(Rng *r, v3 Ve, float Ax, float Ay) {
    float u1 = rng_f(r), u2 = rng_f(r);
    v3 Vh = v3normalize(V3(Ax * Ve.x, Ay * Ve.y, fabsf(Ve.z)));
    float lensq = Vh.x * Vh.x + Vh.y * Vh.y;
    v3 T1 = lensq > 0.0f ? v3scale(V3(-Vh.y, Vh.x, 0.0f), 1.0f / sqrtf(lensq)) : V3(1.0f, 0.0f, 0.0f);
    v3 T2 = v3cross(Vh, T1);
    float rad = sqrtf(u1);
    float phi = 2.0f * ORC_PI * u2;
    float t1 = rad * cosf(phi);
    float t2 = rad * sinf(phi);
    float s = 0.5f * (1.0f + Vh.z);
    t2 = (1.0f - s) * sqrtf(1.0f - t1 * t1) + s * t2;
    v3 Nh = v3add(v3add(v3scale(T1, t1), v3scale(T2, t2)), v3scale(Vh, sqrtf(fmaxf(0.0f, 1.0f - t1 * t1 - t2 * t2))));
    return v3normalize(V3(Ax * Nh.x, Ay * Nh.y, fmaxf(0.0f, Nh.z)));
}
/* SH/Sampler.slang:169-193 */
static inline v3 rng_henyey_greenstein(Rng *r, v3 incident, float G) {
    float rx = rng_f(r), ry = rng_f(r);
    float cosTheta;
    if (fabsf(G) < 1e-5f) {
        cosTheta = 2.0f * rx - 1.0f;
    } else {
        float sqrTerm = (1.0f - G * G) / (1.0f - G + 2.0f * G * rx);
        cosTheta = (1.0f + G * G - sqrTerm * sqrTerm) / (2.0f * G);
    }
    float phi = 2.0f * ORC_PI * ry;
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    v3 nd = V3(sinTheta * cosf(phi), sinTheta * sinf(phi), cosTheta);
    v3 up = fabsf(incident.y) < 0.9999999f ? V3(0, 1, 0) : V3(0, 0, 1);
    v3 tangent = v3normalize(v3cross(up, incident));
    v3 bitangent = v3cross(incident, tangent);
    return v3normalize(v3add(v3add(v3scale(tangent, nd.x), v3scale(bitangent, nd.y)), v3scale(incident, nd.z)));
}

/* ------------------------------------------------------------------------------------------------
 * Scene
 * ---------------------------------------------------------------------------------------------- */
typedef struct { uint32_t mesh, material, tri_count, instance; float transform[16]; } EmissiveEntry; /* PT/PathTracer.h:321-328 */
typedef struct { float o2w[3][4]; float w2o[3][3]; uint32_t tri_base; } InstXf;
typedef struct { v3 v0, v1, v2; uint32_t inst, prim; } WTri;
typedef struct { float lo[3], hi[3]; uint32_t left, right, first, count; } BNode; /* count>0 -> leaf */

struct OrcScene {
    OrcSceneDesc d;
    InstXf *xf;
    EmissiveEntry *emissive; uint32_t n_emissive, n_emissive_tris;
    WTri *tris; uint32_t ntris;
    uint32_t *order;   /* BVH triangle order */
    BNode *nodes; uint32_t nnodes;
};

static v3 xf_point(const float m[3][4], v3 p) {
    return V3(m[0][0] * p.x + m[0][1] * p.y + m[0][2] * p.z + m[0][3] * 1.0f,
              m[1][0] * p.x + m[1][1] * p.y + m[1][2] * p.z + m[1][3] * 1.0f,
              m[2][0] * p.x + m[2][1] * p.y + m[2][2] * p.z + m[2][3] * 1.0f);
}
/* mul(float4x4 M, float4(p,1)).xyz with column-major storage */
static v3 mat4_point(const float t[16], v3 p) {
    return V3(t[0] * p.x + t[4] * p.y + t[8] * p.z + t[12] * 1.0f,
              t[1] * p.x + t[5] * p.y + t[9] * p.z + t[13] * 1.0f,
              t[2] * p.x + t[6] * p.y + t[10] * p.z + t[14] * 1.0f);
}
static v3 mat4_dir(const float t[16], v3 p) { /* w = 0 */
    return V3(t[0] * p.x + t[4] * p.y + t[8] * p.z + t[12] * 0.0f,
              t[1] * p.x + t[5] * p.y + t[9] * p.z + t[13] * 0.0f,
              t[2] * p.x + t[6] * p.y + t[10] * p.z + t[14] * 0.0f);
}
/* mul(n, WorldToObject()).xyz : row-vector times 3x4 -> (W2O^T n) */
static v3 xf_normal(const float w[3][3], v3 n) {
    return V3(n.x * w[0][0] + n.y * w[1][0] + n.z * w[2][0],
              n.x * w[0][1] + n.y * w[1][1] + n.z * w[2][1],
              n.x * w[0][2] + n.y * w[1][2] + n.z * w[2][2]);
}

/* --- BVH (oracle-private: top-down median split, padded boxes) --- */
static void tri_bounds(const WTri *t, float lo[3], float hi[3]) {
    const float *a = &t->v0.x, *b = &t->v1.x, *c = &t->v2.x;
    for (int k = 0; k < 3; k++) { lo[k] = fminf(a[k], fminf(b[k], c[k])); hi[k] = fmaxf(a[k], fmaxf(b[k], c[k])); }
}
static uint32_t bvh_build(OrcScene *s, uint32_t first, uint32_t count) {
    uint32_t id = s->nnodes++;
    BNode *n = &s->nodes[id];
    float lo[3] = { INFINITY, INFINITY, INFINITY }, hi[3] = { -INFINITY, -INFINITY, -INFINITY };
    float clo[3] = { INFINITY, INFINITY, INFINITY }, chi[3] = { -INFINITY, -INFINITY, -INFINITY };
    for (uint32_t i = first; i < first + count; i++) {
        float a[3], b[3]; tri_bounds(&s->tris[s->order[i]], a, b);
        for (int k = 0; k < 3; k++) {
            lo[k] = fminf(lo[k], a[k]); hi[k] = fmaxf(hi[k], b[k]);
            float c = 0.5f * (a[k] + b[k]); clo[k] = fminf(clo[k], c); chi[k] = fmaxf(chi[k], c);
        }
    }
    for (int k = 0; k < 3; k++) { /* conservative padding */
        float pad = 1e-5f * fmaxf(fabsf(lo[k]), fabsf(hi[k])) + 1e-6f;
        n->lo[k] = lo[k] - pad; n->hi[k] = hi[k] + pad;
    }
    n->first = first; n->count = 0; n->left = n->right = 0;
    int axis = 0; float ext = chi[0] - clo[0];
    for (int k = 1; k < 3; k++) if (chi[k] - clo[k] > ext) { ext = chi[k] - clo[k]; axis = k; }
    if (count <= 4 || !(ext > 0.0f)) { n->count = count; return id; }
    float split = 0.5f * (clo[axis] + chi[axis]);
    uint32_t i = first, j = first + count;
    while (i < j) {
        float a[3], b[3]; tri_bounds(&s->tris[s->order[i]], a, b);
        if (0.5f * (a[axis] + b[axis]) < split) i++;
        else { j--; uint32_t tmp = s->order[i]; s->order[i] = s->order[j]; s->order[j] = tmp; }
    }
    uint32_t nl = i - first;
    if (nl == 0 || nl == count) nl = count / 2;
    uint32_t l = bvh_build(s, first, nl);
    uint32_t r = bvh_build(s, first + nl, count - nl);
    s->nodes[id].left = l; s->nodes[id].right = r;
    return id;
}

/* Moeller-Trumbore, no culling.  Accept tmin < t < tmax.  Same formula as the product kernel. */
static inline int tri_hit(const WTri *tr, v3 o, v3 d, float tmin, float tmax, float *t_out, float *u_out, float *v_out) {
    v3 e1 = v3sub(tr->v1, tr->v0), e2 = v3sub(tr->v2, tr->v0);
    v3 p = v3cross(d, e2);
    float det = v3dot(e1, p);
    if (det == 0.0f) return 0;
    float inv = 1.0f / det;
    v3 tv = v3sub(o, tr->v0);
    float u = v3dot(tv, p) * inv;
    if (!(u >= 0.0f && u <= 1.0f)) return 0;
    v3 q = v3cross(tv, e1);
    float v = v3dot(d, q) * inv;
    if (!(v >= 0.0f && u + v <= 1.0f)) return 0;
    float t = v3dot(e2, q) * inv;
    if (!(t > tmin && t < tmax)) return 0;
    *t_out = t; *u_out = u; *v_out = v;
    return 1;
}

typedef struct { int hit; float t, u, v; uint32_t tri; } Hit;

static inline void hit_consider(const OrcScene *s, uint32_t ti, v3 o, v3 d, float tmin, float tmax, Hit *h) {
    float t, u, v;
    if (tri_hit(&s->tris[ti], o, d, tmin, tmax, &t, &u, &v)) {
        if (!h->hit || t < h->t || (t == h->t && ti < h->tri)) { h->hit = 1; h->t = t; h->u = u; h->v = v; h->tri = ti; }
    }
}
static Hit trace_brute(const OrcScene *s, v3 o, v3 d, float tmin, float tmax) {
    Hit h; h.hit = 0; h.t = 0; h.u = h.v = 0; h.tri = 0xFFFFFFFFu;
    for (uint32_t i = 0; i < s->ntris; i++) hit_consider(s, i, o, d, tmin, tmax, &h);
    return h;
}
static Hit trace_bvh(const OrcScene *s, v3 o, v3 d, float tmin, float tmax) {
    Hit h; h.hit = 0; h.t = 0; h.u = h.v = 0; h.tri = 0xFFFFFFFFu;
    if (s->ntris == 0) return h;
    float inv[3] = { 1.0f / d.x, 1.0f / d.y, 1.0f / d.z };
    const float *oo = &o.x;
    uint32_t stack[128]; int sp = 0; stack[sp++] = 0;
    while (sp) {
        const BNode *n = &s->nodes[stack[--sp]];
        float t0 = tmin, t1 = h.hit ? h.t : tmax;
        for (int k = 0; k < 3; k++) {
            float a = (n->lo[k] - oo[k]) * inv[k], b = (n->hi[k] - oo[k]) * inv[k];
            t0 = fmaxf(t0, fminf(a, b)); t1 = fminf(t1, fmaxf(a, b));   /* fminf/fmaxf ignore NaN */
        }
        if (t0 > t1 * 1.0000004f + 1e-30f) continue;
        if (n->count) { for (uint32_t i = 0; i < n->count; i++) hit_consider(s, s->order[n->first + i], o, d, tmin, tmax, &h); }
        else { if (sp < 126) { stack[sp++] = n->left; stack[sp++] = n->right; } }
    }
    return h;
}

OrcScene *orc_scene_create(const OrcSceneDesc *desc) {
    OrcScene *s = (OrcScene *)calloc(1, sizeof(OrcScene));
    s->d = *desc;
    uint32_t ni = desc->ninstances;
    s->xf = (InstXf *)calloc(ni ? ni : 1, sizeof(InstXf));
    s->emissive = (EmissiveEntry *)calloc(ni ? ni : 1, sizeof(EmissiveEntry));
    uint32_t ntris = 0;
    for (uint32_t i = 0; i < ni; i++) {
        const OrcInstance *in = &desc->instances[i];
        InstXf *x = &s->xf[i];
        for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) x->o2w[r][c] = in->transform[c * 4 + r];
        /* inverse of the 3x3 in double, rounded once (driver supplies WorldToObject; SH/Surface.slang:49,60) */
        double m[3][3]; for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) m[r][c] = x->o2w[r][c];
        double det = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
        double id = 1.0 / det;
        x->w2o[0][0] = (float)((m[1][1] * m[2][2] - m[1][2] * m[2][1]) * id);
        x->w2o[0][1] = (float)((m[0][2] * m[2][1] - m[0][1] * m[2][2]) * id);
        x->w2o[0][2] = (float)((m[0][1] * m[1][2] - m[0][2] * m[1][1]) * id);
        x->w2o[1][0] = (float)((m[1][2] * m[2][0] - m[1][0] * m[2][2]) * id);
        x->w2o[1][1] = (float)((m[0][0] * m[2][2] - m[0][2] * m[2][0]) * id);
        x->w2o[1][2] = (float)((m[0][2] * m[1][0] - m[0][0] * m[1][2]) * id);
        x->w2o[2][0] = (float)((m[1][0] * m[2][1] - m[1][1] * m[2][0]) * id);
        x->w2o[2][1] = (float)((m[0][1] * m[2][0] - m[0][0] * m[2][1]) * id);
        x->w2o[2][2] = (float)((m[0][0] * m[1][1] - m[0][1] * m[1][0]) * id);
        x->tri_base = ntris;
        uint32_t tc = desc->meshes[in->mesh].nindices / 3;
        ntris += tc;
        /* emissive list: PT/PathTracer.cpp:458-469 (constant EmissiveColor != 0 only, Q16) */
        const OrcMaterial *mat = &desc->materials[in->material];
        if (mat->EmissiveColor[0] != 0.0f || mat->EmissiveColor[1] != 0.0f || mat->EmissiveColor[2] != 0.0f) {
            EmissiveEntry *e = &s->emissive[s->n_emissive++];
            e->mesh = in->mesh; e->material = in->material; e->tri_count = tc; e->instance = i;
            memcpy(e->transform, in->transform, sizeof(e->transform));
            s->n_emissive_tris += tc;
        }
    }
    s->ntris = ntris;
    s->tris = (WTri *)calloc(ntris ? ntris : 1, sizeof(WTri));
    s->order = (uint32_t *)calloc(ntris ? ntris : 1, sizeof(uint32_t));
    for (uint32_t i = 0; i < ni; i++) {
        const OrcInstance *in = &desc->instances[i];
        const OrcMesh *m = &desc->meshes[in->mesh];
        uint32_t tc = m->nindices / 3;
        for (uint32_t p = 0; p < tc; p++) {
            WTri *t = &s->tris[s->xf[i].tri_base + p];
            const OrcVertex *a = &m->verts[m->indices[p * 3 + 0]], *b = &m->verts[m->indices[p * 3 + 1]], *c = &m->verts[m->indices[p * 3 + 2]];
            t->v0 = xf_point(s->xf[i].o2w, V3(a->pos[0], a->pos[1], a->pos[2]));
            t->v1 = xf_point(s->xf[i].o2w, V3(b->pos[0], b->pos[1], b->pos[2]));
            t->v2 = xf_point(s->xf[i].o2w, V3(c->pos[0], c->pos[1], c->pos[2]));
            t->inst = i; t->prim = p;
        }
    }
    for (uint32_t i = 0; i < ntris; i++) s->order[i] = i;
    s->nodes = (BNode *)calloc(2 * (size_t)(ntris ? ntris : 1) + 2, sizeof(BNode));
    s->nnodes = 0;
    if (ntris) bvh_build(s, 0, ntris);
    return s;
}
void orc_scene_destroy(OrcScene *s) {
    if (!s) return;
    free(s->xf); free(s->emissive); free(s->tris); free(s->order); free(s->nodes); free(s);
}
uint32_t orc_scene_triangle_count(const OrcScene *s) { return s->ntris; }
uint32_t orc_scene_emissive_count(const OrcScene *s) { return s->n_emissive; }
void orc_scene_world_triangles(const OrcScene *s, float *out9, uint32_t *inst_out, uint32_t *prim_out) {
    for (uint32_t i = 0; i < s->ntris; i++) {
        memcpy(out9 + 9 * (size_t)i, &s->tris[i].v0, 9 * sizeof(float));
        if (inst_out) inst_out[i] = s->tris[i].inst;
        if (prim_out) prim_out[i] = s->tris[i].prim;
    }
}
void orc_trace_closest(const OrcScene *s, uint32_t n, const float *org3, const float *dir3, float tmin, float tmax,
                       int use_bvh, float *t_out, uint32_t *prim_out, uint32_t *inst_out, float *uv_out2) {
    for (uint32_t i = 0; i < n; i++) {
        v3 o = V3(org3[3 * i], org3[3 * i + 1], org3[3 * i + 2]), d = V3(dir3[3 * i], dir3[3 * i + 1], dir3[3 * i + 2]);
        Hit h = use_bvh ? trace_bvh(s, o, d, tmin, tmax) : trace_brute(s, o, d, tmin, tmax);
        t_out[i] = h.hit ? h.t : -1.0f;
        prim_out[i] = h.hit ? s->tris[h.tri].prim : 0xFFFFFFFFu;
        inst_out[i] = h.hit ? s->tris[h.tri].inst : 0xFFFFFFFFu;
        if (uv_out2) { uv_out2[2 * i] = h.hit ? h.u : 0.0f; uv_out2[2 * i + 1] = h.hit ? h.v : 0.0f; }
    }
}

/* ------------------------------------------------------------------------------------------------
 * Texture units in software (SURVEY Appendix A): bilinear, texel centres at (i+0.5)/N, no mips.
 * Filtering form: lerp(lerp(t00,t10,a), lerp(t01,t11,a), b) with lerp(p,q,w) = p + w*(q-p).
 * ---------------------------------------------------------------------------------------------- */
static inline float tex_mix(float p, float q, float w) { return p + w * (q - p); }
static inline int wrap_repeat(int i, int n) { int m = i % n; return m < 0 ? m + n : m; }
static inline int clamp_i(int i, int lo, int hi) { return i < lo ? lo : (i > hi ? hi : i); }

/* RGBA8/R8 UNORM texture, REPEAT (PT/PathTracer.cpp:84-91).  R8 returns (r,0,0,1). */
static v4 tex_sample_u8(const OrcTexture *t, float u, float v) {
    int W = (int)t->width, H = (int)t->height, C = (int)t->channels;
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx = floorf(x), fy = floorf(y);
    float ax = x - fx, ay = y - fy;
    int x0 = wrap_repeat((int)fx, W), x1 = wrap_repeat((int)fx + 1, W);
    int y0 = wrap_repeat((int)fy, H), y1 = wrap_repeat((int)fy + 1, H);
    float out[4] = { 0.0f, 0.0f, 0.0f, 1.0f };
    for (int c = 0; c < C; c++) {
        float t00 = (float)t->data[((size_t)y0 * W + x0) * C + c] / 255.0f;
        float t10 = (float)t->data[((size_t)y0 * W + x1) * C + c] / 255.0f;
        float t01 = (float)t->data[((size_t)y1 * W + x0) * C + c] / 255.0f;
        float t11 = (float)t->data[((size_t)y1 * W + x1) * C + c] / 255.0f;
        out[c] = tex_mix(tex_mix(t00, t10, ax), tex_mix(t01, t11, ax), ay);
    }
    v4 r = { out[0], out[1], out[2], out[3] };
    return r;
}
/* RGBA32F env map, REPEAT */
static v4 env_sample(const OrcScene *s, float u, float v) {
    int W = (int)s->d.envW, H = (int)s->d.envH;
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx = floorf(x), fy = floorf(y);
    float ax = x - fx, ay = y - fy;
    int x0 = wrap_repeat((int)fx, W), x1 = wrap_repeat((int)fx + 1, W);
    int y0 = wrap_repeat((int)fy, H), y1 = wrap_repeat((int)fy + 1, H);
    const float *p00 = s->d.env_rgba + ((size_t)y0 * W + x0) * 4, *p10 = s->d.env_rgba + ((size_t)y0 * W + x1) * 4;
    const float *p01 = s->d.env_rgba + ((size_t)y1 * W + x0) * 4, *p11 = s->d.env_rgba + ((size_t)y1 * W + x1) * 4;
    float o[4];
    for (int c = 0; c < 4; c++) o[c] = tex_mix(tex_mix(p00[c], p10[c], ax), tex_mix(p01[c], p11[c], ax), ay);
    v4 r = { o[0], o[1], o[2], o[3] };
    return r;
}
/* R32F 2D-array LUT, CLAMP_TO_EDGE linear in (x,y), nearest (round-half-even) layer (PT/PathTracer.cpp:93-94,871-937) */
static float lut_sample(const float *lut, int W, int H, int L, float u, float v, float layer) {
    int li = clamp_i((int)nearbyintf(layer), 0, L - 1);
    float x = u * (float)W - 0.5f, y = v * (float)H - 0.5f;
    float fx = floorf(x), fy = floorf(y);
    float ax = x - fx, ay = y - fy;
    int x0 = clamp_i((int)fx, 0, W - 1), x1 = clamp_i((int)fx + 1, 0, W - 1);
    int y0 = clamp_i((int)fy, 0, H - 1), y1 = clamp_i((int)fy + 1, 0, H - 1);
    const float *p = lut + (size_t)li * W * H;
    return tex_mix(tex_mix(p[(size_t)y0 * W + x0], p[(size_t)y0 * W + x1], ax),
                   tex_mix(p[(size_t)y1 * W + x0], p[(size_t)y1 * W + x1], ax), ay);
}

/* ------------------------------------------------------------------------------------------------
 * Payload: SH/RTCommon.slang:5-35
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    v3 Origin, Direction, BxDF; float PDF; v3 Emitted;
    uint32_t Depth; Rng Sampler;
    int InMedium; float MediumDensity, MediumAnisotropy; v3 MediumColor, MediumEmissiveColor;
    int VolumeDepth;                                                            /* SH/RTCommon.slang Payload::VolumeDepth, reset per sample (SH/RayGen.slang:61) */
    int ColorChannel;                                                           /* SH/RTCommon.slang:26-29: -1 = all channels, 0/1/2 after an atmosphere event split the ray */
} Payload;

static inline float power_heuristic(float a, float b) { return (a * a) / ((a * a) + (b * b)); } /* SH/RTCommon.slang:124-127 */

/* SH/RTCommon.slang:129-136 */
static inline void direction_to_uv(v3 d, float *u, float *v) {
    float gamma = asinf(d.y);
    float theta = atan2f(d.x, -d.z);
    *u = theta * ORC_1_OVER_PI * 0.5f + 0.5f;
    *v = gamma * ORC_1_OVER_PI + 0.5f;
}

/* ------------------------------------------------------------------------------------------------
 * Surface: SH/Surface.slang:6-159
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    v3 WorldPos; float u, v;
    v3 Normal, Tangent, Bitangent, GeometryNormal;
    v3 P1, P2, P3; /* object-space positions */
    int HitFromInside;
} Surface;

static inline v3 surf_tangent_to_world(const Surface *s, v3 a) {
    return v3normalize(v3add(v3add(v3scale(s->Tangent, a.x), v3scale(s->Bitangent, a.y)), v3scale(s->Normal, a.z)));
}
static inline v3 surf_world_to_tangent(const Surface *s, v3 a) {
    return v3normalize(V3(v3dot(a, s->Tangent), v3dot(a, s->Bitangent), v3dot(a, s->Normal)));
}

static void surface_init(Surface *sf, const OrcScene *sc, const OrcConfig *cfg, uint32_t inst, uint32_t prim,
                         float bu, float bv, v3 rayDir, const OrcTexture *normalTex) {
    const OrcInstance *in = &sc->d.instances[inst];
    const OrcMesh *m = &sc->d.meshes[in->mesh];
    const InstXf *x = &sc->xf[inst];
    float b0 = 1.0f - bu - bv, b1 = bu, b2 = bv;                         /* SH/ClosestHit.slang:45 */
    const OrcVertex *A = &m->verts[m->indices[prim * 3 + 0]], *B = &m->verts[m->indices[prim * 3 + 1]], *C = &m->verts[m->indices[prim * 3 + 2]];
    v3 p1 = V3(A->pos[0], A->pos[1], A->pos[2]), p2 = V3(B->pos[0], B->pos[1], B->pos[2]), p3 = V3(C->pos[0], C->pos[1], C->pos[2]);
    sf->P1 = p1; sf->P2 = p2; sf->P3 = p3;
    v3 lp = v3add(v3add(v3scale(p1, b0), v3scale(p2, b1)), v3scale(p3, b2));  /* :43 */
    sf->WorldPos = xf_point(x->o2w, lp);                                       /* :44 */
    sf->u = A->uv[0] * b0 + B->uv[0] * b1 + C->uv[0] * b2;                    /* :46 */
    sf->v = A->uv[1] * b0 + B->uv[1] * b1 + C->uv[1] * b2;
    v3 gn = v3normalize(v3cross(v3sub(p2, p1), v3sub(p3, p1)));               /* :48 */
    gn = v3normalize(xf_normal(x->w2o, gn));                                   /* :49 */
    v3 n;
    if (cfg->UseOnlyGeometryNormals) {
        n = gn;                                                                /* :53 */
    } else {
        v3 n1 = V3(A->nrm[0], A->nrm[1], A->nrm[2]), n2 = V3(B->nrm[0], B->nrm[1], B->nrm[2]), n3 = V3(C->nrm[0], C->nrm[1], C->nrm[2]);
        n = v3normalize(v3add(v3add(v3scale(n1, b0), v3scale(n2, b1)), v3scale(n3, b2)));   /* :59 */
        n = v3normalize(xf_normal(x->w2o, n));                                 /* :60 */
    }
    v3 view = v3neg(rayDir);                                                   /* :64 */
    if (v3dot(gn, view) < 0.0f) { n = v3neg(n); gn = v3neg(gn); sf->HitFromInside = 1; } else sf->HitFromInside = 0; /* :66-76 */
    v3 up = fabsf(n.z) < 0.9999999f ? V3(0, 0, 1) : V3(1, 0, 0);             /* :78 */
    sf->GeometryNormal = gn;
    sf->Normal = n;
    sf->Tangent = v3normalize(v3cross(up, n));                                 /* :82 */
    sf->Bitangent = v3normalize(v3cross(n, sf->Tangent));                      /* :83 */
    if (!cfg->UseOnlyGeometryNormals) {                                        /* :85-90 (Q10: default map applied too) */
        v4 t = tex_sample_u8(normalTex, sf->u, sf->v);
        v3 nm = V3(t.x * 2.0f - 1.0f, t.y * 2.0f - 1.0f, t.z * 2.0f - 1.0f);
        sf->Normal = surf_tangent_to_world(sf, nm);
    }
    if (v3dot(sf->Normal, view) < 0.0f) {                                      /* :92-100 */
        float eps = 0.01f;
        sf->Normal = v3normalize(v3sub(sf->Normal, v3scale(view, v3dot(sf->Normal, view) - eps)));
    }
    v3 perfect = v3normalize(v3reflect(v3neg(view), sf->Normal));             /* :102 */
    if (v3dot(perfect, gn) < 0.0f) {                                           /* :103-112 */
        float eps = 0.1f;
        float dp = v3dot(sf->Normal, gn);
        sf->Normal = v3normalize(v3add(sf->Normal, v3scale(gn, eps + dp)));
    }
    sf->Tangent = v3normalize(v3cross(sf->Normal, up));                        /* :115 */
    sf->Bitangent = v3normalize(v3cross(sf->Normal, sf->Tangent));             /* :116 */
}
/* SH/Surface.slang:140-147 */
static void surface_rotate_tangents(Surface *sf, float deg) {
    float rot = deg * (ORC_PI / 180.0f);
    float c = cosf(rot), s = sinf(rot);
    v3 T = sf->Tangent, N = sf->Normal;
    v3 r = v3add(v3add(v3scale(T, c), v3scale(v3cross(N, T), s)), v3scale(v3scale(N, v3dot(N, T)), 1.0f - c));
    sf->Tangent = r;
    sf->Bitangent = v3cross(r, N);
}

/* ------------------------------------------------------------------------------------------------
 * Material: SH/Material.slang
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    v3 BaseColor, EmissiveColor, SpecularColor, MediumColor, MediumEmissiveColor;
    float Metallic, Roughness, IOR, Transmission, Anisotropy, AnisotropyRotation, MediumDensity, MediumAnisotropy;
    float Eta, Ax, Ay;
} Mat;
typedef struct { v3 BxDF; float PDF; } Eval;
typedef struct { v3 L; v3 BxDF; float PDF; } BSample;

/* SH/Material.slang:39-87 */
static void material_init(Mat *m, const OrcScene *sc, const OrcConfig *cfg, const OrcMaterial *src, const Surface *sf) {
    m->BaseColor = V3(src->BaseColor[0], src->BaseColor[1], src->BaseColor[2]);
    m->EmissiveColor = V3(src->EmissiveColor[0], src->EmissiveColor[1], src->EmissiveColor[2]);
    m->SpecularColor = V3(src->SpecularColor[0], src->SpecularColor[1], src->SpecularColor[2]);
    m->MediumColor = V3(src->MediumColor[0], src->MediumColor[1], src->MediumColor[2]);
    m->MediumEmissiveColor = V3(src->MediumEmissiveColor[0], src->MediumEmissiveColor[1], src->MediumEmissiveColor[2]);
    m->Metallic = src->Metallic; m->Roughness = src->Roughness; m->IOR = src->IOR; m->Transmission = src->Transmission;
    m->Anisotropy = src->Anisotropy; m->AnisotropyRotation = src->AnisotropyRotation;
    m->MediumDensity = src->MediumDensity; m->MediumAnisotropy = src->MediumAnisotropy;
    v4 tb = tex_sample_u8(&sc->d.textures[src->BaseColorTextureIndex], sf->u, sf->v);
    m->IOR = fmaxf(m->IOR, 1.000001f);
    m->BaseColor = v3mul(m->BaseColor, V3(powf(tb.x, 2.2f), powf(tb.y, 2.2f), powf(tb.z, 2.2f)));
    float tr = tex_sample_u8(&sc->d.textures[src->RoughnessTextureIndex], sf->u, sf->v).x;   /* Q8/Q9 */
    m->Roughness *= tr;
    m->Metallic *= tex_sample_u8(&sc->d.textures[src->MetallicTextureIndex], sf->u, sf->v).x;
    v4 te = tex_sample_u8(&sc->d.textures[src->EmissiveTextureIndex], sf->u, sf->v);
    m->EmissiveColor = v3mul(m->EmissiveColor, V3(te.x, te.y, te.z));
    float aspect = sqrtf(1.0f - sqrtf(m->Anisotropy) * 0.9f);
    m->Ax = fmaxf(0.00001f, m->Roughness / aspect);
    m->Ay = fmaxf(0.00001f, m->Roughness * aspect);
    m->Eta = sf->HitFromInside ? m->IOR : 1.0f / m->IOR;
    if (cfg->FurnaceTestMode) {                                                /* :78-86 */
        m->BaseColor = v3s(1.0f); m->EmissiveColor = v3s(0.0f); m->SpecularColor = v3s(1.0f);
        m->MediumColor = v3s(1.0f); m->MediumEmissiveColor = v3s(0.0f);
    }
}
/* :427-432 */
static inline float schlick_fresnel(float VdotH) { float m = orc_clamp(1.0f - VdotH, 0.0f, 1.0f); float m2 = m * m; return m2 * m2 * m; }
/* :434-449 */
float orc_dielectric_fresnel(float cosI, float eta) {
    float sinT2 = eta * eta * (1.0f - cosI * cosI);
    if (sinT2 > 1.0f) return 1.0f;
    float cosT = sqrtf(fmaxf(1.0f - sinT2, 0.0f));
    float rs = (eta * cosT - cosI) / (eta * cosT + cosI);
    float rp = (eta * cosI - cosT) / (eta * cosI + cosT);
    return 0.5f * (rs * rs + rp * rp);
}
/* :394-404 */
static inline float ggx_d(const Mat *m, v3 H) {
    float Hx2 = H.x * H.x, Hy2 = H.y * H.y, Hz2 = H.z * H.z;
    float ax2 = m->Ax * m->Ax, ay2 = m->Ay * m->Ay;
    float e = Hx2 / ax2 + Hy2 / ay2 + Hz2;
    return 1.0f / (ORC_PI * m->Ax * m->Ay * (e * e));
}
/* :406-423 */
static inline float ggx_lambda(const Mat *m, v3 V) {
    float Vx2 = V.x * V.x, Vy2 = V.y * V.y, Vz2 = fabsf(V.z) * fabsf(V.z);
    float ax2 = m->Ax * m->Ax, ay2 = m->Ay * m->Ay;
    float nom = -1.0f + sqrtf(1.0f + (ax2 * Vx2 + ay2 * Vy2) / Vz2);
    return nom / 2.0f;
}
static inline float ggx_g1(const Mat *m, v3 V) { return 1.0f / (1.0f + ggx_lambda(m, V)); }
/* :331-351 */
static Eval eval_reflection(const Mat *m, v3 V, v3 L, v3 F) {
    Eval e = { V3(0, 0, 0), 0.0f };
    if (L.z <= 1e-5f) return e;
    v3 H = v3normalize(v3add(V, L));
    float VdotH = v3dot(V, H);
    float D = ggx_d(m, H);
    float GV = ggx_g1(m, V), GL = ggx_g1(m, L);
    e.PDF = (GV * fmaxf(VdotH, 0.0f) * D / V.z) / (4.0f * VdotH);
    /* D * F * GV * GL / (4 V.z), left to right */
    e.BxDF = v3divs(v3scale(v3scale(v3scale(F, D), GV), GL), 4.0f * V.z);
    return e;
}
/* :359-387 */
static Eval eval_refraction(const Mat *m, v3 V, v3 L, v3 F) {
    Eval e = { V3(0, 0, 0), 0.0f };
    if (L.z >= 1e-5f) return e;
    v3 H = v3normalize(v3add(v3scale(V, m->Eta), L));
    if (H.z < 0.0f) H = v3neg(H);
    float VdotH = v3dot(V, H), LdotH = v3dot(L, H);
    float D = ggx_d(m, H);
    float GV = ggx_g1(m, V), GL = ggx_g1(m, L);
    float G = GV * GL;
    float den = LdotH + m->Eta * VdotH;
    float den2 = den * den;
    float eta2 = m->Eta * m->Eta;
    float jac = (eta2 * fabsf(LdotH)) / den2;
    e.PDF = (GV * fabsf(VdotH) * D / V.z) * jac;
    /* (F * D * G * eta2 / den2) * (|VdotH| * |LdotH| / |V.z|) */
    float k = fabsf(VdotH) * fabsf(LdotH) / fabsf(V.z);
    e.BxDF = v3scale(v3divs(v3scale(v3scale(v3scale(F, D), G), eta2), den2), k);
    return e;
}
/* :281-289 */
static Eval eval_diffuse(const Mat *m, v3 V, v3 L) {
    (void)V;
    Eval e;
    e.PDF = L.z * ORC_1_OVER_PI;
    e.BxDF = v3scale(v3scale(m->BaseColor, ORC_1_OVER_PI), L.z);
    e.PDF *= (L.z > 0.0f) ? 1.0f : 0.0f;
    return e;
}
/* :291-308 */
static Eval eval_metallic(const Mat *m, const OrcScene *sc, const OrcConfig *cfg, v3 V, v3 L) {
    v3 H = v3normalize(v3add(V, L));
    v3 F = v3lerp(m->BaseColor, m->SpecularColor, schlick_fresnel(v3dot(V, H)));
    Eval e = eval_reflection(m, V, L, F);
    if (cfg->UseEnergyCompensation) {
        float layer = m->Anisotropy * 32.0f;
        float ec = lut_sample(sc->d.lut_reflect, 64, 64, 32, V.z, m->Roughness, layer);
        ec = (1.0f - ec) / ec;
        v3 k = v3add(v3s(1.0f), v3mul(m->BaseColor, v3s(ec)));
        e.BxDF = v3mul(k, e.BxDF);
    }
    return e;
}
/* :310-323 */
static Eval eval_dielectric_reflection(const Mat *m, const OrcScene *sc, const OrcConfig *cfg, v3 V, v3 L) {
    Eval e = eval_reflection(m, V, L, m->SpecularColor);
    if (cfg->UseEnergyCompensation) {
        float layer = m->Anisotropy * 32.0f;
        float ec = lut_sample(sc->d.lut_reflect, 64, 64, 32, V.z, m->Roughness, layer);
        e.BxDF = v3divs(e.BxDF, ec);
    }
    return e;
}
/* :167-279 */
/* :169-177: lobe probabilities */
static void lobe_probs(const Mat *m, float *pm, float *pd, float *pg) {
    *pm = m->Metallic;
    *pd = (1.0f - m->Metallic) * (1.0f - m->Transmission);
    *pg = (1.0f - m->Metallic) * m->Transmission;
    float sum = *pm + *pd + *pg;
    *pm /= sum; *pd /= sum; *pg /= sum;
}
static Eval eval_bsdf(const Mat *m, const OrcScene *sc, const OrcConfig *cfg, v3 V, v3 L) {
    float pm, pd, pg;
    lobe_probs(m, &pm, &pd, &pg);
    int refracted = L.z < 0.0f;
    v3 H; int validRefraction = 0;
    if (refracted) {
        H = v3normalize(v3add(v3scale(V, m->Eta), L));
        if (H.z < 0.0f) H = v3neg(H);
        float VdotH = v3dot(V, H), LdotH = v3dot(L, H);
        validRefraction = (VdotH > 0.0f && LdotH < 0.0f) || (VdotH < 0.0f && LdotH > 0.0f);
    } else {
        H = v3normalize(v3add(V, L));
    }
    float F = orc_dielectric_fresnel(fabsf(v3dot(V, H)), m->Eta);
    Eval out = { V3(0, 0, 0), 0.0f };
    float glassEC = 0.0f;
    if (cfg->UseEnergyCompensation) {
        int inside = m->Eta > 1.0f;
        float layer = (orc_clamp(m->IOR, 1.0001f, 2.0f) - 1.0f) * 32.0f;
        glassEC = lut_sample(inside ? sc->d.lut_refract_in : sc->d.lut_refract_out, 128, 128, 32, sqrtf(V.z), m->Roughness, layer);
    }
    if (!refracted) {
        Eval e = eval_metallic(m, sc, cfg, V, L);
        out.BxDF = v3add(out.BxDF, v3scale(e.BxDF, pm)); out.PDF += e.PDF * pm;
    }
    if (!refracted) {
        Eval e = eval_diffuse(m, V, L);
        out.BxDF = v3add(out.BxDF, v3scale(v3scale(e.BxDF, pd), 1.0f - F)); out.PDF += e.PDF * pd * (1.0f - F);
    }
    if (!refracted) {
        Eval e = eval_dielectric_reflection(m, sc, cfg, V, L);
        out.BxDF = v3add(out.BxDF, v3scale(v3scale(e.BxDF, pd), F)); out.PDF += e.PDF * pd * F;
    }
    if (!refracted) {
        Eval e = eval_reflection(m, V, L, m->SpecularColor);
        if (cfg->UseEnergyCompensation && glassEC > 0.01f) e.BxDF = v3divs(e.BxDF, glassEC);
        out.BxDF = v3add(out.BxDF, v3scale(v3scale(e.BxDF, pg), F)); out.PDF += e.PDF * pg * F;
    }
    if (refracted && validRefraction) {
        Eval e = eval_refraction(m, V, L, m->BaseColor);
        if (cfg->UseEnergyCompensation && glassEC > 0.01f) e.BxDF = v3divs(e.BxDF, glassEC);
        out.BxDF = v3add(out.BxDF, v3scale(v3scale(e.BxDF, pg), 1.0f - F)); out.PDF += e.PDF * pg * (1.0f - F);
    }
    return out;
}
/* :94-165 */
static BSample sample_bsdf(const Mat *m, const OrcScene *sc, const OrcConfig *cfg, Rng *rng, v3 V, v3 H) {
    float pm, pd, pg;
    lobe_probs(m, &pm, &pd, &pg);
    (void)pg;
    float F = orc_dielectric_fresnel(v3dot(V, H), m->Eta);
    float x1 = rng_f(rng);
    v3 L; int refracted = 0;
    if (x1 < pm) {
        L = v3normalize(v3reflect(v3neg(V), H));
    } else if (x1 < pm + pd) {
        if (rng_f(rng) < F) L = v3normalize(v3reflect(v3neg(V), H));
        else L = v3normalize(v3add(rng_sphere(rng), V3(0.0f, 0.0f, 1.0f)));
    } else {
        if (rng_f(rng) < F) L = v3normalize(v3reflect(v3neg(V), H));
        else { L = v3normalize(v3refract(v3neg(V), H, m->Eta)); refracted = 1; }
    }
    BSample z = { V3(0, 0, 0), V3(0, 0, 0), 0.0f };
    if (L.z < 0.0f && !refracted) return z;
    else if (refracted && L.z >= 0.0f) return z;
    Eval e = eval_bsdf(m, sc, cfg, V, L);
    BSample r = { L, e.BxDF, e.PDF };
    return r;
}

/* ------------------------------------------------------------------------------------------------
 * Energy-compensation LUT baker: SH/LookupReflect.slang:25-84, SH/LookupRefract.slang:23-102 (one texel).
 * Not on the render path: it exists so the restated GGX sampler / EvaluateReflection / EvaluateRefraction / DielectricFresnel
 * can be checked against the tables the REFERENCE's own shaders produced (Assets/LookupTables/[*].bin, 10^7 samples/texel).
 * ---------------------------------------------------------------------------------------------- */
float orc_bake_reflect_texel(uint32_t tx, uint32_t ty, uint32_t tz, uint32_t samples, uint32_t seed) {
    const float SX = 64.0f, SY = 64.0f, SZ = 32.0f;                          /* PT/Application.cpp:41 */
    Rng rng = { ty + tx * tx + seed };                                       /* LookupReflect.slang:34 */
    float viewCosine = orc_clamp((float)tx / SX, 0.05f, 0.999f);
    float roughness = orc_clamp((float)ty / SY, 0.0001f, 1.0f);
    float anisotropy = (float)tz / SZ;
    float aspect = sqrtf(1.0f - sqrtf(anisotropy) * 0.9f);
    Mat m; memset(&m, 0, sizeof m);
    m.Anisotropy = anisotropy; m.Roughness = roughness; m.BaseColor = v3s(1.0f);
    m.Ax = fmaxf(0.0001f, roughness / aspect); m.Ay = fmaxf(0.0001f, roughness * aspect);
    double total = 0.0;
    for (uint32_t i = 0; i < samples; i++) {
        float xy = sqrtf(1.0f - viewCosine * viewCosine);
        float phi = rng_f(&rng) * ORC_2PI;
        v3 V = v3normalize(V3(xy * cosf(phi), xy * sinf(phi), viewCosine));
        v3 H = rng_ggx_vndf(&rng, V, m.Ax, m.Ay);
        v3 L = v3normalize(v3reflect(v3neg(V), H));
        if (L.z <= 0.0f) continue;
        Eval e = eval_reflection(&m, V, L, v3s(1.0f));
        if (e.PDF <= 0.0f) continue;
        if (isnan(e.BxDF.x) || isinf(e.BxDF.x)) continue;
        total += e.BxDF.x / e.PDF;
    }
    return (float)(total / samples);
}
/* Exploration hook for the shipped-table study (tests/test_oracle_kat.py): the reflect estimator of
 * LookupReflect.slang:52-82 at explicit parameters, with the two thresholds of the sample loop exposed (reference: lz_min = 0, EvaluateReflection's 1e-5). */
float orc_bake_reflect_params(float viewCosine, float roughness, float anisotropy, float lz_min, uint32_t samples, uint32_t seed) {
    float aspect = sqrtf(1.0f - sqrtf(anisotropy) * 0.9f);
    Mat m; memset(&m, 0, sizeof m);
    m.Anisotropy = anisotropy; m.Roughness = roughness; m.BaseColor = v3s(1.0f);
    m.Ax = fmaxf(0.0001f, roughness / aspect); m.Ay = fmaxf(0.0001f, roughness * aspect);
    Rng rng = { seed };
    double total = 0.0;
    for (uint32_t i = 0; i < samples; i++) {
        float xy = sqrtf(1.0f - viewCosine * viewCosine);
        float phi = rng_f(&rng) * ORC_2PI;
        v3 V = v3normalize(V3(xy * cosf(phi), xy * sinf(phi), viewCosine));
        v3 H = rng_ggx_vndf(&rng, V, m.Ax, m.Ay);
        v3 L = v3normalize(v3reflect(v3neg(V), H));
        if (L.z <= lz_min) continue;
        Eval e = eval_reflection(&m, V, L, v3s(1.0f));
        if (e.PDF <= 0.0f) continue;
        if (isnan(e.BxDF.x) || isinf(e.BxDF.x)) continue;
        total += e.BxDF.x / e.PDF;
    }
    return (float)(total / samples);
}
float orc_bake_refract_texel(uint32_t tx, uint32_t ty, uint32_t tz, int above_surface, uint32_t samples, uint32_t seed) {
    const float SX = 128.0f, SY = 128.0f, SZ = 32.0f;                        /* PT/Application.cpp:54,67 */
    Rng rng = { ty + tx * tx + seed };
    float vc = (float)tx / (SX - 1.0f);
    float viewCosine = orc_clamp(vc * vc, 0.01f, 0.9999f);                   /* LookupRefract.slang:34: pow(.,2) */
    float roughness = orc_clamp((float)ty / (SY - 1.0f), 0.01f, 1.0f);
    float ior = 1.0f + orc_clamp((float)tz / (SZ - 1.0f), 0.0001f, 1.0f);
    Mat m; memset(&m, 0, sizeof m);
    m.Roughness = roughness; m.BaseColor = v3s(1.0f); m.IOR = ior; m.Ax = roughness; m.Ay = roughness;
    m.Eta = above_surface ? (1.0f / ior) : ior;
    double total = 0.0;
    for (uint32_t i = 0; i < samples; i++) {
        float xy = sqrtf(1.0f - viewCosine * viewCosine);
        float phi = rng_f(&rng) * ORC_2PI;
        v3 V = v3normalize(V3(xy * cosf(phi), xy * sinf(phi), viewCosine));
        v3 H = rng_ggx_vndf(&rng, V, m.Ax, m.Ay);
        float F = orc_dielectric_fresnel(fabsf(v3dot(V, H)), m.Eta);
        float val = 0.0f;
        if (rng_f(&rng) < F) {
            v3 L = v3normalize(v3reflect(v3neg(V), H));
            if (L.z > 0.0f) { Eval e = eval_reflection(&m, V, L, v3s(1.0f)); if (e.PDF > 0.0f && !isnan(e.BxDF.x) && !isinf(e.BxDF.x)) val += e.BxDF.x / e.PDF; }
        } else {
            v3 L = v3normalize(v3refract(v3neg(V), H, m.Eta));
            if (L.z < 0.0f) { Eval e = eval_refraction(&m, V, L, v3s(1.0f)); if (e.PDF > 0.0f && !isnan(e.BxDF.x) && !isinf(e.BxDF.x)) val += e.BxDF.x / e.PDF; }
        }
        if (!isnan(val) && !isinf(val)) total += val;
    }
    return (float)(total / samples);
}

/* The whole bake of one texel with the reference's DISPATCH STRUCTURE (PT/LookupTableCalculator.cpp:44-157):
 * loopCount = sampleCount / 20 dispatches of 20 samples; dispatch i re-seeds the per-texel sampler with
 * ty + tx*tx + Seed_i (LookupReflect.slang:30, LookupRefract.slang:32) and does uTable[index] += finalValue / 20 in fp32;
 * the host divides by loopCount at the end (:151-154).  The reference derives Seed_i from the wall clock
 * (PCGHash(i*2 + sampleCount + PCGHash(timeMillis)), :104-105) -- not reproducible -- so `seed` stands in for timeMillis.
 * kind: 0 = LookupReflect, 1 = LookupRefract ABOVE_SURFACE, 2 = LookupRefract BELOW_SURFACE.  Used to check the CUDA baker bit-for-bit. */
float orc_bake_lut_texel(int kind, uint32_t SXu, uint32_t SYu, uint32_t SZu, uint32_t tx, uint32_t ty, uint32_t tz, uint32_t sample_count, uint32_t seed) {
    const float SX = (float)SXu, SY = (float)SYu, SZ = (float)SZu;
    const uint32_t per = 20, loops = sample_count / per;
    Mat m; memset(&m, 0, sizeof m); m.BaseColor = v3s(1.0f);
    float viewCosine;
    if (kind == 0) {
        viewCosine = orc_clamp((float)tx / SX, 0.05f, 0.999f);
        float roughness = orc_clamp((float)ty / SY, 0.0001f, 1.0f), anisotropy = (float)tz / SZ;
        float aspect = sqrtf(1.0f - sqrtf(anisotropy) * 0.9f);
        m.Anisotropy = anisotropy; m.Roughness = roughness;
        m.Ax = fmaxf(0.0001f, roughness / aspect); m.Ay = fmaxf(0.0001f, roughness * aspect);
    } else {
        float vc = (float)tx / (SX - 1.0f);
        viewCosine = orc_clamp(vc * vc, 0.01f, 0.9999f);
        float roughness = orc_clamp((float)ty / (SY - 1.0f), 0.01f, 1.0f);
        float ior = 1.0f + orc_clamp((float)tz / (SZ - 1.0f), 0.0001f, 1.0f);
        m.Roughness = roughness; m.IOR = ior; m.Ax = roughness; m.Ay = roughness;
        m.Eta = kind == 1 ? (1.0f / ior) : ior;
    }
    const uint32_t hseed = orc_pcg_hash(seed);
    float table = 0.0f;
    for (uint32_t i = 0; i < loops; i++) {
        Rng rng = { ty + tx * tx + orc_pcg_hash(i * 2u + sample_count + hseed) };
        float finalValue = 0.0f;
        for (uint32_t k = 0; k < per; k++) {
            float xy = sqrtf(1.0f - viewCosine * viewCosine);
            float phi = rng_f(&rng) * ORC_2PI;
            v3 V = v3normalize(V3(xy * cosf(phi), xy * sinf(phi), viewCosine));
            v3 H = rng_ggx_vndf(&rng, V, m.Ax, m.Ay);
            if (kind == 0) {
                v3 L = v3normalize(v3reflect(v3neg(V), H));
                if (L.z <= 0.0f) continue;
                Eval e = eval_reflection(&m, V, L, v3s(1.0f));
                if (e.PDF <= 0.0f) continue;
                if (isnan(e.BxDF.x) || isinf(e.BxDF.x)) continue;
                finalValue += e.BxDF.x / e.PDF;
            } else {
                float F = orc_dielectric_fresnel(fabsf(v3dot(V, H)), m.Eta);
                float val = 0.0f;
                if (rng_f(&rng) < F) {
                    v3 L = v3normalize(v3reflect(v3neg(V), H));
                    if (L.z > 0.0f) { Eval e = eval_reflection(&m, V, L, v3s(1.0f)); if (e.PDF > 0.0f && !isnan(e.BxDF.x) && !isinf(e.BxDF.x)) val += e.BxDF.x / e.PDF; }
                } else {
                    v3 L = v3normalize(v3refract(v3neg(V), H, m.Eta));
                    if (L.z < 0.0f) { Eval e = eval_refraction(&m, V, L, v3s(1.0f)); if (e.PDF > 0.0f && !isnan(e.BxDF.x) && !isinf(e.BxDF.x)) val += e.BxDF.x / e.PDF; }
                }
                if (!isnan(val) && !isinf(val)) finalValue += val;
            }
        }
        table += finalValue / (float)per;
    }
    return loops ? table / (float)loops : 0.0f;
}

/* ------------------------------------------------------------------------------------------------
 * NEE samplers
 * ---------------------------------------------------------------------------------------------- */
/* SH/Sampler.slang:287-346 */
static void sample_env(const OrcScene *sc, const OrcConfig *cfg, Rng *rng, v3 *toLight, v4 *outValue) {
    float xx = rng_f(rng), xy = rng_f(rng), xz = rng_f(rng);
    uint32_t width = sc->d.envW, height = sc->d.envH;
    uint32_t size = width * height;
    uint32_t idx = (uint32_t)(xx * (float)size); if (idx > size - 1) idx = size - 1;
    OrcAliasEntry e = sc->d.env_alias[idx];
    uint32_t envIdx;
    if (xy < e.Importance) { envIdx = idx; xy /= e.Importance; }
    else { envIdx = e.Alias; xy = (xy - e.Importance) / (1.0f - e.Importance); }
    uint32_t px = envIdx % width, py = envIdx / width;
    float u = ((float)px + xy) / (float)width;
    float phi = u * (2.0f * ORC_PI) - ORC_PI;
    float sinPhi = sinf(phi), cosPhi = cosf(phi);
    float stepTheta = ORC_PI / (float)height;
    float theta0 = (float)py * stepTheta;
    float cosTheta = cosf(theta0) * (1.0f - xz) + cosf(theta0 + stepTheta) * xz;
    float theta = acosf(cosTheta);
    float sinTheta = sinf(theta);
    float v = theta * ORC_1_OVER_PI;
    v3 d = V3(sinPhi * sinTheta, -cosTheta, -cosPhi * sinTheta);
    float az = cfg->SkyRotationAzimuth / 180.0f * ORC_PI;
    float al = cfg->SkyRotationAltitude / 180.0f * ORC_PI;
    d = orc_rotate(d, V3(0, 1, 0), az);
    d = orc_rotate(d, V3(1, 0, 0), al);
    *toLight = d;
    v4 val = env_sample(sc, u, v);
    val.x *= cfg->EnvironmentIntensity; val.y *= cfg->EnvironmentIntensity; val.z *= cfg->EnvironmentIntensity;
    *outValue = val;
}
/* SH/Sampler.slang:349-422 */
static void sample_emissive(const OrcScene *sc, Rng *rng, v3 pos, v3 *toLight, v4 *colorPDF, uint32_t *tri, uint32_t *inst) {
    *tri = 0xFFFFFFFFu; *inst = 0xFFFFFFFFu;
    uint32_t count = sc->n_emissive;
    if (count == 0) { *toLight = V3(0, 0, 0); v4 z = { 0, 0, 0, 0 }; *colorPDF = z; return; }
    uint32_t mi = (uint32_t)floorf(rng_f(rng) * (float)count); if (mi > count - 1) mi = count - 1;
    const EmissiveEntry *em = &sc->emissive[mi];
    *inst = em->instance;
    uint32_t ti = (uint32_t)floorf(rng_f(rng) * (float)em->tri_count); if (ti > em->tri_count - 1) ti = em->tri_count - 1;
    *tri = ti;
    const OrcMesh *m = &sc->d.meshes[em->mesh];
    const OrcVertex *A = &m->verts[m->indices[ti * 3 + 0]], *B = &m->verts[m->indices[ti * 3 + 1]], *C = &m->verts[m->indices[ti * 3 + 2]];
    v3 p0 = mat4_point(em->transform, V3(A->pos[0], A->pos[1], A->pos[2]));
    v3 p1 = mat4_point(em->transform, V3(B->pos[0], B->pos[1], B->pos[2]));
    v3 p2 = mat4_point(em->transform, V3(C->pos[0], C->pos[1], C->pos[2]));
    float x0 = rng_f(rng), x1 = rng_f(rng);
    float su1 = sqrtf(x0);
    float b0 = 1.0f - su1, b1 = x1 * su1, b2 = 1.0f - b0 - b1;
    v3 tp = v3add(v3add(v3scale(p0, b0), v3scale(p1, b1)), v3scale(p2, b2));
    float uu = b0 * A->uv[0] + b1 * B->uv[0] + b2 * C->uv[0];
    float vv = b0 * A->uv[1] + b1 * B->uv[1] + b2 * C->uv[1];
    v3 dlt = v3sub(tp, pos);
    *toLight = v3normalize(dlt);
    v3 normal = v3normalize(v3cross(v3sub(p2, p0), v3sub(p1, p0)));
    float area = v3length(v3cross(v3sub(p1, p0), v3sub(p2, p0))) * 0.5f;
    float d2 = v3dot(dlt, dlt);
    float cosTheta = fabsf(v3dot(normal, *toLight));
    const OrcMaterial *mat = &sc->d.materials[em->material];
    v4 te = tex_sample_u8(&sc->d.textures[mat->EmissiveTextureIndex], uu, vv);
    v4 r;
    r.w = d2 / ((float)count * (float)em->tri_count * area * cosTheta);
    r.x = mat->EmissiveColor[0] * te.x; r.y = mat->EmissiveColor[1] * te.y; r.z = mat->EmissiveColor[2] * te.z;
    *colorPDF = r;
}

/* SH/RTCommon.slang:47-84 (USE_RAY_QUERIES variant, the default PT/PathTracer.h:218) */
static int does_ray_intersect(const OrcScene *sc, v3 o, v3 d, uint32_t *tri, uint32_t *inst, uint64_t *shadow_rays) {
    *tri = 0; *inst = 0;
    (*shadow_rays)++;
    Hit h = trace_bvh(sc, o, d, 0.0001f, 1000000.0f);
    if (h.hit) { *tri = sc->tris[h.tri].prim; *inst = sc->tris[h.tri].inst; return 1; }
    return 0;
}

/* ------------------------------------------------------------------------------------------------
 * Homogeneous AABB volumes: SH/Volume.slang (the m_DensityDataIndex == -1 paths), SH/RayGen.slang:162-380,
 * phase functions SH/RTCommon.slang:214-227 and their samplers SH/Sampler.slang:169-284.
 * ---------------------------------------------------------------------------------------------- */
typedef struct { float Near, Far; } VolIsect;
/* SH/Volume.slang:188-211 (the y/z mix-up of the max/min chains is the reference's) */
static VolIsect vol_intersect(v3 o, v3 d, const float mn[3], const float mx[3]) {
    v3 inv = V3(1.0f / d.x, 1.0f / d.y, 1.0f / d.z);
    v3 t0 = v3mul(v3sub(V3(mn[0], mn[1], mn[2]), o), inv), t1 = v3mul(v3sub(V3(mx[0], mx[1], mx[2]), o), inv);
    v3 ts = V3(fminf(t0.x, t1.x), fminf(t0.y, t1.y), fminf(t0.z, t1.z)), tb = V3(fmaxf(t0.x, t1.x), fmaxf(t0.y, t1.y), fmaxf(t0.z, t1.z));
    float tmin = fmaxf(fmaxf(ts.x, ts.y), fmaxf(ts.x, ts.z));
    float tmax = fminf(fminf(tb.x, tb.y), fminf(tb.x, tb.z));
    VolIsect r = { tmin, tmax };
    if (tmax < 0.0f || tmin > tmax) { r.Near = -1.0f; r.Far = -1.0f; }
    return r;
}
/* SH/Volume.slang:150-156 */
static float vol_effective_anisotropy(const OrcVolume *v, float rayDepth) {
    if (v->ApproximatedScattering != 0) {
        float sg = v->Anisotropy > 0.0f ? 1.0f : (v->Anisotropy < 0.0f ? -1.0f : 0.0f);
        return powf(fabsf(v->Anisotropy), 1.0f + rayDepth) * sg;
    }
    return v->Anisotropy;
}
/* SH/RTCommon.slang:214-221 */
static float phase_hg(v3 V, v3 L, float g) {
    if (g == 0.0f) return 1.0f / (4.0f * ORC_PI);
    float c = v3dot(V, L);
    return (1.0f / (4.0f * ORC_PI)) * ((1.0f - g * g) / powf(1.0f + g * g - 2.0f * g * c, 1.5f));
}
/* SH/RTCommon.slang:223-228 */
static float phase_draine(v3 V, v3 L, float g, float a) {
    float c = v3dot(V, L);
    return ((1.0f - g * g) * (1.0f + a * c * c)) / (4.0f * (1.0f + (a * (1.0f + 2.0f * g * g)) / 3.0f) * ORC_PI * powf(1.0f + g * g - 2.0f * g * c, 1.5f));
}
/* rotation of a tangent-space direction around the incident direction, shared tail of SH/Sampler.slang:183-192 / :265-274 */
static v3 phase_frame(v3 incident, float cosTheta, float phi) {
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    v3 nd = V3(sinTheta * cosf(phi), sinTheta * sinf(phi), cosTheta);
    v3 up = fabsf(incident.y) < 0.9999999f ? V3(0, 1, 0) : V3(0, 0, 1);
    v3 tangent = v3normalize(v3cross(up, incident));
    v3 bitangent = v3cross(incident, tangent);
    return v3normalize(v3add(v3add(v3scale(tangent, nd.x), v3scale(bitangent, nd.y)), v3scale(incident, nd.z)));
}
/* SH/Sampler.slang:219-276 */
static v3 rng_draine(Rng *r, v3 incident, float g, float a) {
    float rx = rng_f(r), ry = rng_f(r);
    float cosTheta;
    if (fabsf(g) < 1e-5f) {
        cosTheta = 2.0f * rx - 1.0f;
    } else if (fabsf(a) < 1e-5f) {
        float sqrTerm = (1.0f - g * g) / (1.0f - g + 2.0f * g * rx);
        cosTheta = (1.0f + g * g - sqrTerm * sqrTerm) / (2.0f * g);
    } else {
        const float g2 = g * g, g3 = g * g2, g4 = g2 * g2, g6 = g2 * g4;
        const float pgp1_2 = (1.0f + g2) * (1.0f + g2);
        const float T1a = -a + a * g4;
        const float T1a3 = T1a * T1a * T1a;
        const float T2 = -1296.0f * (-1.0f + g2) * (a - a * g2) * (T1a) * (4.0f * g2 + a * pgp1_2);
        const float T3 = 3.0f * g2 * (1.0f + g * (-1.0f + 2.0f * rx)) + a * (2.0f + g2 + g3 * (1.0f + 2.0f * g2) * (-1.0f + 2.0f * rx));
        const float T4a = 432.0f * T1a3 + T2 + 432.0f * (a - a * g2) * T3 * T3;
        const float T4b = -144.0f * a * g2 + 288.0f * a * g4 - 144.0f * a * g6;
        const float T4b3 = T4b * T4b * T4b;
        const float T4 = T4a + sqrtf(-4.0f * T4b3 + T4a * T4a);
        const float T4p3 = powf(T4, 1.0f / 3.0f);
        const float cbrt2 = powf(2.0f, 1.0f / 3.0f);
        const float T6 = (2.0f * T1a + (48.0f * cbrt2 * (-(a * g2) + 2.0f * a * g4 - a * g6)) / T4p3 + T4p3 / (3.0f * cbrt2)) / (a - a * g2);
        const float T5 = 6.0f * (1.0f + g2) + T6;
        const float q = -0.5f * sqrtf(T5) + sqrtf(6.0f * (1.0f + g2) - (8.0f * T3) / (a * (-1.0f + g2) * sqrtf(T5)) - T6) / 2.0f;
        cosTheta = (1.0f + g2 - q * q) / (2.0f * g);
    }
    return phase_frame(incident, cosTheta, 2.0f * ORC_PI * ry);
}
/* Conditioning study of the Draine inversion above (tests/test_oracle_kat.py::test_draine_inversion_is_ill_conditioned_in_fp32): the SAME
 * expression tree evaluated in fp32 (what the shader, this oracle and the CUDA kernel do) and in fp64.  T4a and sqrt(-4 T4b^3 + T4a^2) are
 * of magnitude 1e3..1e9 and nearly cancel, so the fp32 value of cos(theta) carries an error far above one ulp: two correct fp32 implementations
 * that round differently (FMA contraction, libm) disagree on the scattered direction by more than 1e-4 in a few per cent of the draws. */
#define DRAINE_COS(T, SQRT, POW, rx, g, a, out) do {                                                                              \
        const T g2 = g * g, g3 = g * g2, g4 = g2 * g2, g6 = g2 * g4;                                                              \
        const T pgp1_2 = ((T)1 + g2) * ((T)1 + g2);                                                                               \
        const T T1a = -a + a * g4;                                                                                                \
        const T T1a3 = T1a * T1a * T1a;                                                                                           \
        const T T2 = (T)-1296 * ((T)-1 + g2) * (a - a * g2) * (T1a) * ((T)4 * g2 + a * pgp1_2);                                    \
        const T T3 = (T)3 * g2 * ((T)1 + g * ((T)-1 + (T)2 * rx)) + a * ((T)2 + g2 + g3 * ((T)1 + (T)2 * g2) * ((T)-1 + (T)2 * rx)); \
        const T T4a = (T)432 * T1a3 + T2 + (T)432 * (a - a * g2) * T3 * T3;                                                       \
        const T T4b = (T)-144 * a * g2 + (T)288 * a * g4 - (T)144 * a * g6;                                                       \
        const T T4b3 = T4b * T4b * T4b;                                                                                           \
        const T T4 = T4a + SQRT((T)-4 * T4b3 + T4a * T4a);                                                                        \
        const T T4p3 = POW(T4, (T)1 / (T)3);                                                                                      \
        const T cbrt2 = POW((T)2, (T)1 / (T)3);                                                                                   \
        const T T6 = ((T)2 * T1a + ((T)48 * cbrt2 * (-(a * g2) + (T)2 * a * g4 - a * g6)) / T4p3 + T4p3 / ((T)3 * cbrt2)) / (a - a * g2); \
        const T T5 = (T)6 * ((T)1 + g2) + T6;                                                                                     \
        const T q = (T)-0.5 * SQRT(T5) + SQRT((T)6 * ((T)1 + g2) - ((T)8 * T3) / (a * ((T)-1 + g2) * SQRT(T5)) - T6) / (T)2;       \
        out = ((T)1 + g2 - q * q) / ((T)2 * g);                                                                                    \
    } while (0)
void orc_draine_cos_theta(float rx, float g, float a, float *cos32, double *cos64) {
    float c32; DRAINE_COS(float, sqrtf, powf, rx, g, a, c32);
    const double rxd = rx, gd = g, ad = a; double c64; DRAINE_COS(double, sqrt, pow, rxd, gd, ad, c64);
    *cos32 = c32; *cos64 = c64;
}
/* droplet-size fit of SH/Volume.slang:389-400 / SH/Sampler.slang:278-295 */
static void hg_draine_fit(float d, float *GHG, float *GD, float *ALPHA_D, float *W_D) {
    *GHG = expf(-(0.0990567f / (d - 1.67154f)));
    *GD = expf(-(2.20679f / (d + 3.91029f)) - 0.428934f);
    *ALPHA_D = expf(3.62489f - (8.29288f / (d + 5.52825f)));
    *W_D = expf(-(0.599085f / (d - 0.641583f)) - 0.665888f);
}
/* Volume::GetScatteringDirection, SH/Volume.slang:354-371 */
static v3 vol_scatter_direction(const OrcConfig *cfg, const OrcVolume *v, Rng *rng, v3 incident, int rayDepth) {
    if (cfg->PhaseFunction == 0) return rng_henyey_greenstein(rng, incident, vol_effective_anisotropy(v, (float)rayDepth));
    if (cfg->PhaseFunction == 1) return rng_draine(rng, incident, vol_effective_anisotropy(v, (float)rayDepth), v->Alpha);
    float GHG, GD, AD, WD; hg_draine_fit(v->DropletSize, &GHG, &GD, &AD, &WD);          /* SH/Sampler.slang:278-295 */
    GHG = powf(fmaxf(GHG, 0.0f), 1.0f + (float)rayDepth);
    GD = powf(fmaxf(GD, 0.0f), 1.0f + (float)rayDepth);
    float u = rng_f(rng);
    if (u < WD) return rng_henyey_greenstein(rng, incident, GHG);
    return rng_draine(rng, incident, GD, AD);
}
/* Volume::EvaluatePhaseFunction, SH/Volume.slang:373-401 (the HG+Draine evaluation ignores the depth, unlike its sampler) */
static float vol_phase(const OrcConfig *cfg, const OrcVolume *v, v3 V, v3 L, int rayDepth) {
    if (cfg->PhaseFunction == 0) return phase_hg(V, L, vol_effective_anisotropy(v, (float)rayDepth));
    if (cfg->PhaseFunction == 1) return phase_draine(V, L, vol_effective_anisotropy(v, (float)rayDepth), v->Alpha);
    float GHG, GD, AD, WD; hg_draine_fit(v->DropletSize, &GHG, &GD, &AD, &WD);
    return orc_lerp(phase_hg(V, L, GHG), phase_draine(V, L, GD, AD), WD);
}
/* ---- heterogeneous volumes: SH/Volume.slang:54-166,230-252,291-352,448-517 over OrcGrid (the dense restatement of the NanoVDB reads, pt_oracle.h) ---- */
#define GRID_DIM 32                                                              /* MAX_DENSITY_GRID_DIM, SH/Volume.slang:11 */
/* SampleNanoVDBBuffer, SH/Volume.slang:69-117: three raw PCG draws jitter the voxel */
static float grid_sample(const OrcVolume *v, const OrcGrid *g, Rng *rng, v3 x) {
    float minX = (float)g->WorldBBox[0], minY = (float)g->WorldBBox[1], minZ = (float)g->WorldBBox[2];
    float maxX = (float)g->WorldBBox[3], maxY = (float)g->WorldBBox[4], maxZ = (float)g->WorldBBox[5];
    int wmin[3] = { (int)floorf(minX), (int)floorf(minY), (int)floorf(minZ) }, wmax[3] = { (int)ceilf(maxX), (int)ceilf(maxY), (int)ceilf(maxZ) };
    v3 np = V3((x.x - v->CornerMin[0]) / (v->CornerMax[0] - v->CornerMin[0]), (x.y - v->CornerMin[1]) / (v->CornerMax[1] - v->CornerMin[1]),
               (x.z - v->CornerMin[2]) / (v->CornerMax[2] - v->CornerMin[2]));
    np.y = 1.0f - np.y;                                                          /* :83 */
    v3 gp = V3(np.x * (float)(wmax[0] - wmin[0]) + (float)wmin[0], np.y * (float)(wmax[1] - wmin[1]) + (float)wmin[1], np.z * (float)(wmax[2] - wmin[2]) + (float)wmin[2]);
    /* pnanovdb_grid_world_to_indexf: (src - vecf) * invmatf (diagonal map), then pnanovdb_hdda_pos_to_ijk: floor */
    v3 ip = V3((gp.x - g->Translation[0]) * g->InvVoxelSize[0], (gp.y - g->Translation[1]) * g->InvVoxelSize[1], (gp.z - g->Translation[2]) * g->InvVoxelSize[2]);
    int c[3] = { (int)floorf(ip.x), (int)floorf(ip.y), (int)floorf(ip.z) };
    c[0] = (int)((uint32_t)c[0] + (rng_pcg(rng) % 3u - 1u));                     /* :103-105 (unsigned wrap-around = -1 / 0 / +1) */
    c[1] = (int)((uint32_t)c[1] + (rng_pcg(rng) % 3u - 1u));
    c[2] = (int)((uint32_t)c[2] + (rng_pcg(rng) % 3u - 1u));
    for (int k = 0; k < 3; k++) {                                                /* :108 clamp to the root bbox */
        int lo = g->IndexMin[k], hi = g->IndexMin[k] + (int)g->Dim[k] - 1;
        c[k] = c[k] < lo ? lo : (c[k] > hi ? hi : c[k]);
    }
    float value = g->Values[((size_t)(c[2] - g->IndexMin[2]) * g->Dim[1] + (size_t)(c[1] - g->IndexMin[1])) * g->Dim[0] + (size_t)(c[0] - g->IndexMin[0])];
    return orc_clamp(value / v->MaxDensityInTheGrid * v->GridSharpness, 0.0f, 1.0f);   /* :116 */
}
static float vol_effective_density(const OrcVolume *v, float baseDensity, float rayDepth) {     /* :159-166 */
    if (v->ApproximatedScattering != 0) return baseDensity * powf(v->ApproximatedScatteringFalloff, rayDepth);
    return baseDensity;
}
typedef struct { v3 blockSize; float epsilon, tEnter, tExit; } VolCtx;
typedef struct { int blockIndex; v3 minCorner, maxCorner; } VolBlock;
static VolCtx vol_ctx(const OrcVolume *v, VolIsect is) {                         /* CreateTraversalContext, :119-128 */
    VolCtx c;
    v3 ext = V3(v->CornerMax[0] - v->CornerMin[0], v->CornerMax[1] - v->CornerMin[1], v->CornerMax[2] - v->CornerMin[2]);
    c.blockSize = V3(ext.x / (float)GRID_DIM, ext.y / (float)GRID_DIM, ext.z / (float)GRID_DIM);
    c.epsilon = 0.0001f * fmaxf(ext.x, fmaxf(ext.y, ext.z));
    c.tEnter = fmaxf(is.Near, 0.0f); c.tExit = is.Far;
    return c;
}
static VolBlock vol_block(const OrcVolume *v, v3 p, const VolCtx *c) {           /* CalculateBlockInfo, :131-147 */
    VolBlock b;
    v3 rel = V3((p.x - v->CornerMin[0]) / (v->CornerMax[0] - v->CornerMin[0]), (p.y - v->CornerMin[1]) / (v->CornerMax[1] - v->CornerMin[1]),
                (p.z - v->CornerMin[2]) / (v->CornerMax[2] - v->CornerMin[2]));
    int ix = (int)(rel.x * (float)GRID_DIM), iy = (int)(rel.y * (float)GRID_DIM), iz = (int)(rel.z * (float)GRID_DIM);
    ix = ix < 0 ? 0 : (ix > GRID_DIM - 1 ? GRID_DIM - 1 : ix); iy = iy < 0 ? 0 : (iy > GRID_DIM - 1 ? GRID_DIM - 1 : iy); iz = iz < 0 ? 0 : (iz > GRID_DIM - 1 ? GRID_DIM - 1 : iz);
    b.blockIndex = ix + iy * GRID_DIM + iz * GRID_DIM * GRID_DIM;
    b.minCorner = V3(v->CornerMin[0] + c->blockSize.x * (float)ix, v->CornerMin[1] + c->blockSize.y * (float)iy, v->CornerMin[2] + c->blockSize.z * (float)iz);
    b.maxCorner = v3add(b.minCorner, c->blockSize);
    return b;
}
static VolIsect vol_intersect_v(v3 o, v3 d, v3 mn, v3 mx) { float a[3] = { mn.x, mn.y, mn.z }, b[3] = { mx.x, mx.y, mx.z }; return vol_intersect(o, d, a, b); }
/* ProcessHeterogeneousVolumeScattering, SH/Volume.slang:291-352: delta tracking against the per-block majorants */
static float vol_scatter_distance_grid(const OrcVolume *v, const OrcGrid *g, v3 o, v3 d, Rng *rng, float rayDepth, VolIsect is) {
    VolCtx c = vol_ctx(v, is);
    VolBlock b = vol_block(v, v3add(o, v3scale(d, c.tEnter + c.epsilon)), &c);
    float t = 0.0f;
    for (int i = 0; i < 10000; i++) {
        v3 cur = v3add(o, v3scale(d, c.tEnter + t + c.epsilon));
        VolIsect bi = vol_intersect_v(cur, d, b.minCorner, b.maxCorner);
        float maxDensity = vol_effective_density(v, g->MaxDensities[b.blockIndex] * v->Density, rayDepth);
        float sampled = -logf(rng_f(rng)) / maxDensity;
        if (bi.Far <= 0.0f) {
            t += c.epsilon;
            if (c.tEnter + t > c.tExit) return -1.0f;
            b = vol_block(v, v3add(o, v3scale(d, c.tEnter + t + c.epsilon)), &c);
            continue;
        }
        float toExit = bi.Far - fmaxf(bi.Near, 0.0f);
        if (sampled > toExit) {
            t += toExit + c.epsilon;
            if (c.tEnter + t > c.tExit) return -1.0f;
            b = vol_block(v, v3add(o, v3scale(d, c.tEnter + t + c.epsilon)), &c);
            continue;
        }
        t += sampled;
        if (c.tEnter + t > c.tExit) return -1.0f;
        v3 sp = v3add(o, v3scale(d, c.tEnter + t));
        float dens = vol_effective_density(v, grid_sample(v, g, rng, sp) * v->Density, rayDepth);
        if (dens / maxDensity < rng_f(rng)) continue;                            /* null collision */
        return c.tEnter + t;
    }
    return -1.0f;
}
/* ProcessHeterogeneousVolumeTransmittance, SH/Volume.slang:448-517: ratio tracking with Russian roulette */
static float vol_transmittance_grid(const OrcVolume *v, const OrcGrid *g, Rng *rng, v3 o, v3 d, float rayDepth, VolIsect is) {
    VolCtx c = vol_ctx(v, is);
    VolBlock b = vol_block(v, v3add(o, v3scale(d, c.tEnter + c.epsilon)), &c);
    float T = 1.0f, t = 0.0f;
    for (int j = 0; j < 1000; j++) {
        v3 cur = v3add(o, v3scale(d, c.tEnter + t + c.epsilon));
        VolIsect bi = vol_intersect_v(cur, d, b.minCorner, b.maxCorner);
        float maxDensity = vol_effective_density(v, g->MaxDensities[b.blockIndex] * v->Density, rayDepth);
        float sampled = -logf(rng_f(rng)) / maxDensity;
        if (bi.Far <= 0.0f) {
            t += c.epsilon;
            if (c.tEnter + t > c.tExit) break;
            b = vol_block(v, v3add(o, v3scale(d, c.tEnter + t + c.epsilon)), &c);
            continue;
        }
        float toExit = bi.Far - fmaxf(bi.Near, 0.0f);
        if (sampled > toExit) {
            t += toExit + c.epsilon;
            if (c.tEnter + t > c.tExit) break;
            b = vol_block(v, v3add(o, v3scale(d, c.tEnter + t + c.epsilon)), &c);
            continue;
        }
        t += sampled;
        if (c.tEnter + t > c.tExit) break;
        v3 ip = v3add(o, v3scale(d, c.tEnter + t));
        float dens = vol_effective_density(v, grid_sample(v, g, rng, ip) * v->Density, rayDepth);
        T *= 1.0f - (dens / maxDensity);
        float p = T;
        if (rng_f(rng) > p) return 0.0f;
        T /= p;
    }
    return T;
}
/* Volume::CalculateVolumesTransmittance, SH/Volume.slang:419-446: analytic for homogeneous volumes, a random walk (on the payload's sampler) for
 * each heterogeneous volume the ray crosses */
static float volumes_transmittance(const OrcConfig *cfg, Rng *rng, v3 o, v3 d, float rayDepth) {
    float T = 1.0f;
    for (uint32_t i = 0; i < cfg->VolumesCount; i++) {
        const OrcVolume *v = &cfg->Volumes[i];
        VolIsect is = vol_intersect(o, d, v->CornerMin, v->CornerMax);
        is.Near = fmaxf(is.Near, 0.0f);
        if (v->DensityDataIndex >= 0 && is.Far >= 0.0f) {
            T *= vol_transmittance_grid(v, &cfg->Grids[v->DensityDataIndex], rng, o, d, rayDepth, is);
            if (T <= 0.0f) return 0.0f;
        } else {
            float len = is.Far - is.Near;
            if (len > 0.0f) T *= expf(-v->Density * len);
        }
    }
    return orc_clamp(T, 0.0f, 1.0f);
}
/* Volume::DoesRayScatterInVolume, SH/Volume.slang:254-289 (homogeneous branch: one random number when the ray crosses the box) */
static float vol_scatter_distance(const OrcConfig *cfg, const OrcVolume *v, v3 o, v3 d, Rng *rng, float rayDepth, float ignoreIfFartherThan) {
    VolIsect is = vol_intersect(o, d, v->CornerMin, v->CornerMax);
    if (is.Far < 0.0f) return -1.0f;
    if (ignoreIfFartherThan >= 0.0f && is.Near > ignoreIfFartherThan) return -1.0f;
    float inside = is.Far - fmaxf(is.Near, 0.0f);
    if (inside <= 0.0f) return -1.0f;
    if (v->DensityDataIndex >= 0) return vol_scatter_distance_grid(v, &cfg->Grids[v->DensityDataIndex], o, d, rng, rayDepth, is);
    float sampled = -logf(rng_f(rng)) / v->Density;                             /* SH/Sampler.slang:425-428 */
    if (sampled < inside) return fmaxf(is.Near, 0.0f) + sampled;
    return -1.0f;
}
/* Blackbody, SH/RTCommon.slang:139-172 */
static v3 blackbody(float temperature) {
    float temp = temperature / 100.0f;
    float r, g, b;
    if (temp <= 66.0f) r = 255.0f; else r = 329.698727446f * powf(temp - 60.0f, -0.1332047592f);
    if (temp <= 66.0f) g = 99.4708025861f * logf(temp) - 161.1195681661f; else g = 288.1221695283f * powf(temp - 60.0f, -0.0755148492f);
    if (temp >= 66.0f) b = 255.0f; else if (temp <= 19.0f) b = 0.0f; else b = 138.5177312231f * logf(temp - 10.0f) - 305.0447927307f;
    return V3(orc_clamp(r / 255.0f, 0.0f, 1.0f), orc_clamp(g / 255.0f, 0.0f, 1.0f), orc_clamp(b / 255.0f, 0.0f, 1.0f));
}
/* Volume::GetEmissionFromTemperatureAtPoint, SH/Volume.slang:230-252: the temperature is read from the DENSITY buffer (:235) */
static v3 vol_temperature_emission(const OrcConfig *cfg, const OrcVolume *v, Rng *rng, v3 x) {
    if (!v->HasTemperatureData) return v3s(0.0f);
    float tn = grid_sample(v, &cfg->Grids[v->DensityDataIndex], rng, x);
    v3 color;
    if (v->UseBlackbody) color = blackbody(tn * (float)(v->KelvinMax - v->KelvinMin) + (float)v->KelvinMin);
    else color = V3(v->TemperatureColor[0], v->TemperatureColor[1], v->TemperatureColor[2]);
    float intensity = powf(tn, v->TemperatureGamma) * v->TemperatureScale;
    return V3(intensity * powf(color.x, v->EmissiveColorGamma), intensity * powf(color.y, v->EmissiveColorGamma), intensity * powf(color.z, v->EmissiveColorGamma));
}
static int does_ray_intersect(const OrcScene *sc, v3 o, v3 d, uint32_t *tri, uint32_t *inst, uint64_t *shadow_rays);
static void sample_env(const OrcScene *sc, const OrcConfig *cfg, Rng *rng, v3 *toLight, v4 *outValue);
static void sample_emissive(const OrcScene *sc, Rng *rng, v3 pos, v3 *toLight, v4 *colorPDF, uint32_t *tri, uint32_t *inst);
static void importance_sample_sky(const OrcScene *sc, const OrcConfig *cfg, Rng *rng, v3 *toLight, v4 *outValue);
static v3 atm_transmittance_nee(const OrcConfig *c, Payload *pl, v3 ro, v3 rd);
/* EvaluateVolumeScatteringEvent, SH/RayGen.slang:265-380 */
static void volume_scatter_event(const OrcScene *sc, const OrcConfig *cfg, Payload *pl, float scatterDistance, int vi, OrcCounters *cnt) {
    const OrcVolume *v = &cfg->Volumes[vi];
    const v3 color = V3(v->Color[0], v->Color[1], v->Color[2]);
    pl->Origin = v3add(pl->Origin, v3scale(pl->Direction, scatterDistance));
    pl->Emitted = v3add(V3(v->EmissiveColor[0], v->EmissiveColor[1], v->EmissiveColor[2]), vol_temperature_emission(cfg, v, &pl->Sampler, pl->Origin));   /* :268 */
    v3 toSky = V3(0, 0, 0); v4 sky = { 0, 0, 0, 0 };
    if (cfg->EnableSkyMIS) {
        importance_sample_sky(sc, cfg, &pl->Sampler, &toSky, &sky);
        sky.x *= cfg->EnvironmentIntensity; sky.y *= cfg->EnvironmentIntensity; sky.z *= cfg->EnvironmentIntensity;   /* :277 (Q7 again) */
        uint32_t t0, t1;
        if (does_ray_intersect(sc, pl->Origin, toSky, &t0, &t1, &cnt->shadow_rays)) { v4 z = { 0, 0, 0, 0 }; sky = z; }
    }
    v3 toLight = V3(0, 0, 0); v4 light = { 0, 0, 0, 0 };
    if (cfg->EnableMeshMIS) {
        uint32_t lt, li, ht, hi;
        sample_emissive(sc, &pl->Sampler, pl->Origin, &toLight, &light, &lt, &li);
        does_ray_intersect(sc, pl->Origin, toLight, &ht, &hi, &cnt->shadow_rays);       /* a miss leaves (0, 0): compared all the same, :301-302 */
        if (ht != lt || hi != li) { v4 z = { 0, 0, 0, 0 }; light = z; }
    }
    const v3 newDir = vol_scatter_direction(cfg, v, &pl->Sampler, pl->Direction, pl->VolumeDepth);
    const float phaseS = vol_phase(cfg, v, pl->Direction, newDir, pl->VolumeDepth);
    if (cfg->EnableSkyMIS && sky.w > 0.0f) {
        float ph = vol_phase(cfg, v, pl->Direction, toSky, pl->VolumeDepth);
        v3 T = v3s(volumes_transmittance(cfg, &pl->Sampler, pl->Origin, toSky, (float)pl->VolumeDepth));      /* :326 */
        if (cfg->EnableAtmosphere) T = v3mul(T, atm_transmittance_nee(cfg, pl, pl->Origin, toSky));   /* :328-342 */
        v3 bx = v3scale(color, ph);
        if (ph > 0.0f)
            pl->Emitted = v3add(pl->Emitted, v3scale(v3mul(v3mul(T, bx), v3divs(V3(sky.x, sky.y, sky.z), sky.w)), power_heuristic(sky.w, ph)));
    }
    if (cfg->EnableMeshMIS && light.w > 0.0f) {
        float ph = vol_phase(cfg, v, pl->Direction, toLight, pl->VolumeDepth);
        float T = volumes_transmittance(cfg, &pl->Sampler, pl->Origin, toLight, (float)(pl->VolumeDepth + 1));   /* :361 */
        v3 bx = v3scale(color, ph);
        if (ph > 0.0f)
            pl->Emitted = v3add(pl->Emitted, v3scale(v3mul(v3mul(v3s(T), bx), v3divs(V3(light.x, light.y, light.z), light.w)), power_heuristic(light.w, ph)));
    }
    pl->Direction = newDir;
    pl->BxDF = v3scale(color, phaseS);
    pl->PDF = phaseS;
    pl->Depth++;
    pl->VolumeDepth++;
    cnt->medium_events++;
}
static Hit trace_bvh(const OrcScene *s, v3 o, v3 d, float tmin, float tmax);

/* ------------------------------------------------------------------------------------------------
 * Atmosphere (ENABLE_ATMOSPHERE): SH/Atmosphere.slang, SH/RayGen.slang:382-471, SH/Sampler.slang:196-215,430-476, SH/RTCommon.slang:174-211
 * ---------------------------------------------------------------------------------------------- */
static const float ATM_C_RAYLEIGH[3] = { 5.802f * 1e-6f, 13.558f * 1e-6f, 33.100f * 1e-6f };        /* Atmosphere.slang:7 */
static const float ATM_C_MIE_SCATTERING = 3.996f * 1e-6f, ATM_C_MIE_ABSORPTION = 4.40f * 1e-6f;    /* :8-9 */
static const float ATM_C_OZONE[3] = { 0.650f * 1e-6f, 1.881f * 1e-6f, 0.085f * 1e-6f };             /* :11 */
typedef struct { float x, y; } v2;
static v2 intersect_sphere(v3 ro, v3 rd, v3 center, float radius) {                                  /* RTCommon.slang:174-193 */
    ro = v3sub(ro, center);
    float a = v3dot(rd, rd);
    float b = 2.0f * v3dot(ro, rd);
    float c = v3dot(ro, ro) - radius * radius;
    float disc = b * b - 4.0f * a * c;
    v2 r = { -1.0f, -1.0f };
    if (disc < 0.0f) return r;
    r.x = (-b - sqrtf(disc)) / (2.0f * a);
    r.y = (-b + sqrtf(disc)) / (2.0f * a);
    return r;
}
static inline v3 atm_planet(const OrcConfig *c) { return V3(c->PlanetPosition[0], c->PlanetPosition[1], c->PlanetPosition[2]); }
static float atm_height(const OrcConfig *c, v3 p) { return v3length(v3sub(p, atm_planet(c))) - c->PlanetRadius; }   /* Atmosphere.slang:13-16 */
static float atm_rayleigh_density(const OrcConfig *c, float h) { return expf(-h / c->RayleighDensityFalloff); }
static float atm_mie_density(const OrcConfig *c, float h) { return expf(-h / c->MieDensityFalloff); }
static float atm_ozone_density(const OrcConfig *c, float h) { return expf(-(fabsf(h - c->OzonePeak) / c->OzoneDensityFalloff)); }
static void atm_coefficients(const OrcConfig *c, int ch, float *kr, float *km, float *ko) {
    const float C_MIE = ATM_C_MIE_SCATTERING + ATM_C_MIE_ABSORPTION;                                 /* :10 */
    *kr = ATM_C_RAYLEIGH[ch] * c->RayleighScatteringCoefficientMultiplier[ch];
    *km = C_MIE * c->MieScatteringCoefficientMultiplier[ch];
    *ko = ATM_C_OZONE[ch] * c->OzoneAbsorptionCoefficientMultiplier[ch];
}
/* CalculateTransmittanceThroughAtmosphere, Atmosphere.slang:33-104: ratio tracking with Russian roulette on ONE colour channel; returns a
 * vector that is zero in the other two channels */
static v3 atm_transmittance(const OrcConfig *c, Rng *rng, v3 ro, v3 rd, int ch) {
    v2 pi = intersect_sphere(ro, rd, atm_planet(c), c->PlanetRadius);
    if (pi.y > 0.0f) return v3s(0.0f);                                                               /* occluded by the planet */
    v2 ai = intersect_sphere(ro, rd, atm_planet(c), c->PlanetRadius + c->AtmosphereHeight);
    float tMin = fmaxf(ai.x, 0.0f), tMax = ai.y;
    if (tMax < 0.0f) return v3s(1.0f);
    float kr, km, ko; atm_coefficients(c, ch, &kr, &km, &ko);
    float majorant = atm_rayleigh_density(c, 0.0f) * kr + atm_mie_density(c, 0.0f) * km + atm_ozone_density(c, c->OzonePeak) * ko;
    if (majorant <= 0.0f) return v3s(1.0f);
    float t = 0.0f, T = 1.0f;
    for (int i = 0; i < 1000; i++) {
        float deltaT = -logf(1.0f - rng_f(rng)) / majorant;
        t += deltaT;
        if (t >= tMax - tMin) break;
        float h = atm_height(c, v3add(ro, v3scale(rd, t + tMin)));
        if (h < 0.0f) break;
        float dr = atm_rayleigh_density(c, h) * kr, dm = atm_mie_density(c, h) * km, dz = atm_ozone_density(c, h) * ko;
        T *= 1.0f - (dr + dm + dz) / majorant;
        float p = T;
        if (rng_f(rng) > p) { T = 0.0f; break; }
        T /= p;
    }
    v3 out = v3s(0.0f);
    if (ch == 0) out.x = T; else if (ch == 1) out.y = T; else out.z = T;
    return out;
}
/* the NEE transmittance of SH/ClosestHit.slang:335-349 / SH/RayGen.slang:328-342: three walks while the ray is unsplit, one after */
static v3 atm_transmittance_nee(const OrcConfig *c, Payload *pl, v3 ro, v3 rd) {
    if (pl->ColorChannel == -1) {
        v3 T;
        T.x = atm_transmittance(c, &pl->Sampler, ro, rd, 0).x;
        T.y = atm_transmittance(c, &pl->Sampler, ro, rd, 1).y;
        T.z = atm_transmittance(c, &pl->Sampler, ro, rd, 2).z;
        return T;
    }
    return atm_transmittance(c, &pl->Sampler, ro, rd, pl->ColorChannel);
}
/* SampleAtmosphereScatterDistance, Atmosphere.slang:114-201: delta tracking; *component: -1 none, 0 Rayleigh, 1 Mie, 2 ozone */
static float atm_sample_scatter_distance(const OrcConfig *c, Rng *rng, v3 ro, v3 rd, int ch, int *component) {
    v2 ai = intersect_sphere(ro, rd, atm_planet(c), c->PlanetRadius + c->AtmosphereHeight);
    float tMinA = fmaxf(ai.x, 0.0f), tMaxA = ai.y;
    *component = -1;
    v2 pi = intersect_sphere(ro, rd, atm_planet(c), c->PlanetRadius);
    float tMinPlanet = pi.x;
    if (tMaxA < 0.0f) return -1.0f;
    float kr, km, ko; atm_coefficients(c, ch, &kr, &km, &ko);
    float majorant = atm_rayleigh_density(c, 0.0f) * kr + atm_mie_density(c, 0.0f) * km + atm_ozone_density(c, c->OzonePeak) * ko;
    if (majorant <= 0.0f) return -1.0f;
    float t = tMinA;
    for (int i = 0; i < 1000; i++) {
        float deltaT = -logf(1.0f - rng_f(rng)) / majorant;
        t += deltaT;
        if (t >= tMaxA) break;
        if (tMinPlanet > 0.0f && t >= tMinPlanet) break;
        float h = atm_height(c, v3add(ro, v3scale(rd, t)));
        float dr = atm_rayleigh_density(c, h) * kr, dm = atm_mie_density(c, h) * km, dz = atm_ozone_density(c, h) * ko;
        float density = dr + dm + dz;
        if (density / majorant < rng_f(rng)) continue;                                               /* null collision */
        float pr = dr / density, pm = dm / density;
        float x = rng_f(rng);
        if (x <= pr) *component = 0; else if (x <= pr + pm) *component = 1; else *component = 2;
        return t;
    }
    return -1.0f;
}
static float phase_rayleigh(v3 V, v3 L) { float ct = v3dot(V, L); return (3.0f / (16.0f * ORC_PI)) * (1.0f + ct * ct); }   /* RTCommon.slang:197-201 */
static float phase_mie_approx(v3 V, v3 L, float g) {                                                 /* RTCommon.slang:204-211 */
    float ct = v3dot(V, L);
    g = fminf(g, 0.9381f);
    float k = 1.55f * g - 0.55f * g * g * g;
    float kc = k * ct;
    return (1.0f - k * k) / ((4.0f * ORC_PI) * (1.0f - kc) * (1.0f - kc));
}
static float phase_hg(v3 V, v3 L, float g);
static v3 phase_frame(v3 incident, float cosTheta, float phi);
static v3 rng_rayleigh(Rng *r, v3 incident) {                                                        /* Sampler.slang:196-215 */
    float rx = rng_f(r), ry = rng_f(r);
    float a = 2.0f * rx - 1.0f;
    float u = -powf(2.0f * a + sqrtf(4.0f * powf(a, 2.0f) + 1.0f), 1.0f / 3.0f);
    float cosTheta = u - (1.0f / u);
    return phase_frame(incident, cosTheta, 2.0f * ORC_PI * ry);
}
/* SampleSunDisk(0.004675), Sampler.slang:430-463 (ImportanceSampleSky with ENABLE_ATMOSPHERE, :465-476) */
static void sample_sun_disk(const OrcConfig *c, Rng *rng, v3 *toLight, v4 *colorPDF) {
    const float sunTheta = 0.004675f;
    float az = c->SkyRotationAzimuth / 180.0f * ORC_PI, al = c->SkyRotationAltitude / 180.0f * ORC_PI;
    v3 sunDir = orc_rotate(V3(0.0f, 0.0f, -1.0f), V3(1.0f, 0.0f, 0.0f), al);
    sunDir = orc_rotate(sunDir, V3(0.0f, 1.0f, 0.0f), az);
    float cosThetaMax = cosf(sunTheta);
    float phi = 2.0f * ORC_PI * rng_f(rng);
    float cosTheta = orc_lerp(cosThetaMax, 1.0f, rng_f(rng));
    float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
    v3 local = V3(cosf(phi) * sinTheta, sinf(phi) * sinTheta, cosTheta);
    v3 w = v3normalize(sunDir);
    v3 up = fabsf(w.z) < 0.999f ? V3(0, 0, 1) : V3(1, 0, 0);
    v3 u = v3normalize(v3cross(up, w));
    v3 v = v3cross(w, u);
    *toLight = v3add(v3add(v3scale(u, local.x), v3scale(v, local.y)), v3scale(w, local.z));
    float solidAngle = 2.0f * ORC_PI * (1.0f - cosThetaMax);
    colorPDF->w = 1.0f / solidAngle;
    colorPDF->x = 2e5f * c->SunColor[0] * c->EnvironmentIntensity; colorPDF->y = 2e5f * c->SunColor[1] * c->EnvironmentIntensity; colorPDF->z = 2e5f * c->SunColor[2] * c->EnvironmentIntensity;
}
static void sample_env(const OrcScene *sc, const OrcConfig *cfg, Rng *rng, v3 *toLight, v4 *outValue);
static void importance_sample_sky(const OrcScene *sc, const OrcConfig *cfg, Rng *rng, v3 *toLight, v4 *outValue) {   /* Sampler.slang:465-476 */
    if (cfg->EnableAtmosphere) sample_sun_disk(cfg, rng, toLight, outValue);
    else sample_env(sc, cfg, rng, toLight, outValue);
}
static int does_ray_intersect(const OrcScene *sc, v3 o, v3 d, uint32_t *tri, uint32_t *inst, uint64_t *shadow_rays);
static float volumes_transmittance(const OrcConfig *cfg, Rng *rng, v3 o, v3 d, float rayDepth);
/* EvaluateAtmosphereScatteringEvent, SH/RayGen.slang:382-471 */
static void atmosphere_scatter_event(const OrcScene *sc, const OrcConfig *cfg, Payload *pl, float scatterDistance, int component, OrcCounters *cnt) {
    pl->Origin = v3add(pl->Origin, v3scale(pl->Direction, scatterDistance));
    v3 newDir;
    if (component == 0) newDir = rng_rayleigh(&pl->Sampler, pl->Direction);
    else if (component == 1) newDir = rng_henyey_greenstein(&pl->Sampler, pl->Direction, 0.85f);
    else newDir = pl->Direction;                                                                     /* ozone only absorbs */
    const float C_MIE = ATM_C_MIE_SCATTERING + ATM_C_MIE_ABSORPTION;
    if (cfg->EnableSkyMIS) {
        v3 toSun; v4 cp;
        importance_sample_sky(sc, cfg, &pl->Sampler, &toSun, &cp);
        cp.x *= cfg->EnvironmentIntensity; cp.y *= cfg->EnvironmentIntensity; cp.z *= cfg->EnvironmentIntensity;
        uint32_t t0, t1;
        int obscured = does_ray_intersect(sc, pl->Origin, toSun, &t0, &t1, &cnt->shadow_rays);
        v3 T = v3s(0.0f);
        if (!obscured) {
            T = atm_transmittance(cfg, &pl->Sampler, pl->Origin, toSun, pl->ColorChannel);
            T = v3scale(T, volumes_transmittance(cfg, &pl->Sampler, pl->Origin, toSun, (float)pl->VolumeDepth));   /* :421 */
        }
        v3 col = v3divs(V3(cp.x, cp.y, cp.z), cp.w);
        if (component == 0) {
            float ph = phase_rayleigh(pl->Direction, toSun);
            pl->Emitted = v3add(pl->Emitted, v3mul(v3scale(T, ph), col));
            float pn = phase_rayleigh(pl->Direction, newDir);
            pl->BxDF = v3s(pn); pl->PDF = pn;
        } else if (component == 1) {
            float ph = phase_hg(pl->Direction, toSun, 0.85f);
            pl->Emitted = v3add(pl->Emitted, v3mul(v3scale(T, ph), col));
            float att = ATM_C_MIE_ABSORPTION / C_MIE;
            float pn = phase_hg(pl->Direction, newDir, 0.85f);
            pl->BxDF = v3s(pn * (1.0f - att)); pl->PDF = pn;
        } else { pl->BxDF = v3s(0.0f); pl->PDF = 1.0f; }
    } else {
        if (component == 0) { float pn = phase_rayleigh(pl->Direction, newDir); pl->BxDF = v3s(pn); pl->PDF = pn; }
        else { float att = ATM_C_MIE_ABSORPTION / C_MIE; pl->BxDF = v3s(phase_mie_approx(pl->Direction, newDir, 0.85f) * att); pl->PDF = phase_hg(pl->Direction, newDir, 0.85f); }
    }
    pl->Direction = newDir;
    pl->Depth++;
    cnt->medium_events++;
}

/* ScatteredInVolume, SH/RayGen.slang:162-263 */
#define ORC_MAX_VOLUMES 100
static int scattered_in_volume(const OrcScene *sc, const OrcConfig *cfg, Payload *pl, OrcCounters *cnt) {
    float distances[ORC_MAX_VOLUMES]; int indices[ORC_MAX_VOLUMES];
    const int n = (int)(cfg->VolumesCount < ORC_MAX_VOLUMES ? cfg->VolumesCount : ORC_MAX_VOLUMES);
    for (int i = 0; i < n; i++) {
        VolIsect is = vol_intersect(pl->Origin, pl->Direction, cfg->Volumes[i].CornerMin, cfg->Volumes[i].CornerMax);
        distances[i] = fmaxf(0.0f, is.Near); indices[i] = i;
    }
    for (int i = 0; i < n; i++)
        for (int j = i + 1; j < n; j++)
            if (distances[j] < distances[i]) { float td = distances[i]; int ti = indices[i]; distances[i] = distances[j]; indices[i] = indices[j]; distances[j] = td; indices[j] = ti; }
    /* GetDistanceToGeometry, SH/RTCommon.slang:86-100: un-normalised direction, tmin 1e-5, tmax 1e6 */
    Hit gh = trace_bvh(sc, pl->Origin, pl->Direction, 0.00001f, 1000000.0f);
    const float distanceToGeometry = gh.hit ? gh.t : -1.0f;
    float scatterDistance = -1.0f; int scattered = -1;
    for (int i = 0; i < n; i++) {
        float t = vol_scatter_distance(cfg, &cfg->Volumes[indices[i]], pl->Origin, pl->Direction, &pl->Sampler, (float)pl->Depth, scatterDistance);   /* :199: payload.Depth, not VolumeDepth */
        if (t >= 0.0f && (t < scatterDistance || scatterDistance < 0.0f)) { scatterDistance = t; scattered = indices[i]; }
    }
    int component = -1, colorChannel = pl->ColorChannel;
    if (cfg->EnableAtmosphere) {                                                 /* :212-236 */
        if (colorChannel == -1) {
            float pick = rng_f(&pl->Sampler);
            colorChannel = pick < 0.33333f ? 0 : (pick < 0.66666f ? 1 : 2);
        }
        float ta = atm_sample_scatter_distance(cfg, &pl->Sampler, pl->Origin, pl->Direction, colorChannel, &component);
        if (ta >= 0.0f && (ta < scatterDistance || scatterDistance < 0.0f)) { scatterDistance = ta; scattered = -2; }
    }
    if (scatterDistance >= 0.0f && (distanceToGeometry < 0.0f || scatterDistance < distanceToGeometry)) {
        if (scattered == -2) { pl->ColorChannel = colorChannel; atmosphere_scatter_event(sc, cfg, pl, scatterDistance, component, cnt); }
        else volume_scatter_event(sc, cfg, pl, scatterDistance, scattered, cnt);
        return 1;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------------
 * ClosestHit: SH/ClosestHit.slang:20-378
 * ---------------------------------------------------------------------------------------------- */
/* The parts of closest_hit that orc_shade_query runs too, so that the render path and the query path cannot drift apart. */
/* :40-67: surface, material, isLight, rotated tangents */
static int hit_surface(const OrcScene *sc, const OrcConfig *cfg, uint32_t inst, uint32_t prim, float bu, float bv, v3 rayDir, Surface *sf, Mat *m) {
    const OrcMaterial *cm = &sc->d.materials[sc->d.instances[inst].material];
    surface_init(sf, sc, cfg, inst, prim, bu, bv, rayDir, &sc->d.textures[cm->NormalTextureIndex]);
    material_init(m, sc, cfg, cm, sf);
    int isLight = m->EmissiveColor.x > 0.0f || m->EmissiveColor.y > 0.0f || m->EmissiveColor.z > 0.0f;  /* :65 */
    surface_rotate_tangents(sf, m->AnisotropyRotation);                        /* :67 */
    return isLight;
}
/* BSDF sampling :191-204: V in tangent space, the VNDF half vector and the sampled direction */
static BSample hit_sample_bsdf(const OrcScene *sc, const OrcConfig *cfg, const Surface *sf, const Mat *m, Rng *rng, v3 rayDir, v3 *V, v3 *H) {
    *V = surf_world_to_tangent(sf, v3normalize(v3neg(rayDir)));
    *H = rng_ggx_vndf(rng, *V, m->Ax, m->Ay);
    return sample_bsdf(m, sc, cfg, rng, *V, *H);
}
/* emission :265-317 of a hit at Depth `depth` reached from `origin` with BSDF pdf `pdf` */
static v3 hit_emission(const OrcScene *sc, const OrcConfig *cfg, uint32_t inst, const Surface *sf, const Mat *m, int isLight, uint32_t depth, v3 origin, float pdf) {
    v3 e = V3(0, 0, 0);
    if (cfg->EnableMeshMIS) {
        if (depth == 0 && isLight) {
            e = v3add(e, m->EmissiveColor);
        } else if (isLight) {
            v3 w1 = xf_point(sc->xf[inst].o2w, sf->P1), w2 = xf_point(sc->xf[inst].o2w, sf->P2), w3 = xf_point(sc->xf[inst].o2w, sf->P3);
            float area = v3length(v3cross(v3sub(w2, w1), v3sub(w3, w1))) * 0.5f;
            v3 dl = v3sub(sf->WorldPos, origin);
            float d2 = v3dot(dl, dl);
            float cosTheta = fabsf(v3dot(sf->Normal, v3normalize(v3sub(origin, sf->WorldPos))));
            uint32_t triCount = 0;
            for (uint32_t i = 0; i < sc->n_emissive; i++) if (sc->emissive[i].instance == inst) { triCount = sc->emissive[i].tri_count; break; }
            float lp = (1.0f / (float)sc->n_emissive) * (1.0f / (float)triCount) * (1.0f / area) * (d2 / cosTheta);
            lp = fmaxf(lp, cfg->EmissiveMeshSamplingPDFBias);
            e = v3add(e, v3scale(m->EmissiveColor, power_heuristic(pdf, lp)));
        }
    } else {
        e = v3add(e, m->EmissiveColor);
    }
    return e;
}
/* sky draw :125-131: direction (world, and returned in tangent space) and radiance | pdf, radiance scaled once more by the intensity (Q7) */
static v3 hit_sky_draw(const OrcScene *sc, const OrcConfig *cfg, const Surface *sf, Rng *rng, v3 *toSkyW, v4 *sky) {
    importance_sample_sky(sc, cfg, rng, toSkyW, sky);
    sky->x *= cfg->EnvironmentIntensity; sky->y *= cfg->EnvironmentIntensity; sky->z *= cfg->EnvironmentIntensity;
    return surf_world_to_tangent(sf, *toSkyW);
}
/* one NEE term :341-344, :366-369: BxDF * T * radiance / pdf, MIS-weighted */
static v3 nee_term(Eval e, v3 T, v4 lv) {
    v3 c = v3divs(v3mul(v3mul(e.BxDF, T), V3(lv.x, lv.y, lv.z)), lv.w);
    return v3scale(c, power_heuristic(lv.w, e.PDF));
}

static void closest_hit(const OrcScene *sc, const OrcConfig *cfg, Payload *pl, v3 rayDir, const Hit *h, OrcCounters *cnt) {
    pl->Emitted = V3(0, 0, 0);                                                  /* :24 */
    uint32_t inst = sc->tris[h->tri].inst, prim = sc->tris[h->tri].prim;
    Surface sf;
    Mat m;
    int isLight = hit_surface(sc, cfg, inst, prim, h->u, h->v, rayDir, &sf, &m);

    if (pl->InMedium) {                                                         /* :80-116 (Q6) */
        float dist = v3length(v3sub(pl->Origin, sf.WorldPos));
        if (pl->MediumAnisotropy == 1.0f) {
            v3 a = v3scale(v3scale(v3neg(v3sub(v3s(1.0f), m.MediumColor)), m.MediumDensity), dist);
            pl->BxDF = V3(expf(a.x), expf(a.y), expf(a.z));
        } else {
            float sd = -logf(rng_f(&pl->Sampler)) / pl->MediumDensity;
            if (sd < dist) {
                pl->Origin = v3add(pl->Origin, v3scale(pl->Direction, sd));
                pl->Direction = rng_henyey_greenstein(&pl->Sampler, pl->Direction, pl->MediumAnisotropy);
                pl->BxDF = pl->MediumColor;
                cnt->medium_events++;
                return;
            }
        }
    }
    cnt->surface_hits++;

    /* sky NEE :125-147 */
    v3 toSkyW = V3(0, 0, 0), toSkyT = V3(0, 0, 0); v4 sky = { 0, 0, 0, 0 }; int canHitSky = 0;
    if (cfg->EnableSkyMIS) {
        toSkyT = hit_sky_draw(sc, cfg, &sf, &pl->Sampler, &toSkyW, &sky);
        uint32_t t0, t1;
        canHitSky = !does_ray_intersect(sc, v3add(sf.WorldPos, v3scale(sf.Normal, 1e-5f)), toSkyW, &t0, &t1, &cnt->shadow_rays);
        if (!canHitSky) { v4 z = { 0, 0, 0, 0 }; sky = z; }
    }
    /* light NEE :154-184 */
    v3 toLightW = V3(0, 0, 0), toLightT = V3(0, 0, 0); v4 light = { 0, 0, 0, 0 }; int canHitLight = 0;
    if (cfg->EnableMeshMIS && !isLight) {
        uint32_t lt, li;
        sample_emissive(sc, &pl->Sampler, sf.WorldPos, &toLightW, &light, &lt, &li);
        if (light.w > 0.0f) {
            toLightT = surf_world_to_tangent(&sf, toLightW);
            uint32_t ht, hi;
            int found = does_ray_intersect(sc, v3add(sf.WorldPos, v3scale(toLightW, 1e-2f)), toLightW, &ht, &hi, &cnt->shadow_rays);
            canHitLight = found ? (lt == ht && li == hi) : 0;
            if (!canHitLight) { v4 z = { 0, 0, 0, 0 }; light = z; }
        }
    }
    v3 V, H;
    BSample ss = hit_sample_bsdf(sc, cfg, &sf, &m, &pl->Sampler, rayDir, &V, &H);
    int wasRefracted = ss.L.z < 0.0f;
    v3 scatterW = surf_tangent_to_world(&sf, ss.L);
    if (!wasRefracted && v3dot(scatterW, sf.GeometryNormal) < 0.0f) { ss.PDF = 0.0f; ss.BxDF = V3(0, 0, 0); }   /* :220-225 */
    if (wasRefracted && sf.HitFromInside) {                                     /* :227-238 */
        pl->InMedium = 0;
    } else if (wasRefracted && !sf.HitFromInside) {
        pl->InMedium = 1;
        pl->MediumColor = m.MediumColor; pl->MediumEmissiveColor = m.MediumEmissiveColor;
        pl->MediumAnisotropy = m.MediumAnisotropy; pl->MediumDensity = m.MediumDensity;
    }
    Eval skyEval = { V3(0, 0, 0), 0.0f };
    if (cfg->EnableSkyMIS && canHitSky) skyEval = eval_bsdf(&m, sc, cfg, V, toSkyT);          /* :241-247 */
    Eval lightEval = { V3(0, 0, 0), 0.0f };
    if (cfg->EnableMeshMIS && canHitLight && !isLight) lightEval = eval_bsdf(&m, sc, cfg, V, toLightT); /* :250-256 */

    pl->Emitted = v3add(pl->Emitted, hit_emission(sc, cfg, inst, &sf, &m, isLight, pl->Depth, pl->Origin, pl->PDF));   /* :265-317 */
    /* payload write :319-324 */
    float off = -1e-3f * (wasRefracted ? 1.0f : 0.0f) + 1e-3f * (wasRefracted ? 0.0f : 1.0f);
    pl->Origin = v3add(sf.WorldPos, v3scale(sf.Normal, off));
    pl->Direction = scatterW;
    pl->BxDF = ss.BxDF;
    pl->PDF = ss.PDF;
    /* NEE accumulation :326-372 (volume transmittance == 1 with VolumesCount == 0, SH/Volume.slang:419-446) */
    if (cfg->EnableSkyMIS && canHitSky) {
        v3 T = v3s(cfg->VolumesCount ? volumes_transmittance(cfg, &pl->Sampler, pl->Origin, toSkyW, 0.0f) : 1.0f);     /* :332-333 */
        if (cfg->EnableAtmosphere) T = v3mul(T, atm_transmittance_nee(cfg, pl, pl->Origin, toSkyW));    /* :335-349: consumes random numbers whenever the sky is visible */
        if (sky.w > 0.0f && skyEval.PDF > 0.0f) pl->Emitted = v3add(pl->Emitted, nee_term(skyEval, T, sky));
    }
    if (cfg->EnableMeshMIS && !isLight && canHitLight && light.w > 0.0f && lightEval.PDF > 0.0f) {
        const float T = cfg->VolumesCount ? volumes_transmittance(cfg, &pl->Sampler, pl->Origin, toLightW, 0.0f) : 1.0f;    /* :364 */
        pl->Emitted = v3add(pl->Emitted, nee_term(lightEval, v3s(T), light));
    }
    int invalid = ss.PDF <= 0.0f;                                               /* :375-376 */
    pl->Depth = ORC_MAX_DEPTH * (invalid ? 1u : 0u) + (pl->Depth + 1u * (invalid ? 0u : 1u));
}

/* One hit's shading step (pt_oracle.h): closest_hit's draws in its order, without the shadow rays, at Depth 1 outside any medium. */
static void put3(float *o, v3 a) { o[0] = a.x; o[1] = a.y; o[2] = a.z; }
static void put_eval(float *o, Eval e) { put3(o, e.BxDF); o[3] = e.PDF; }
static void put_bits(float *o, uint32_t u) { memcpy(o, &u, 4); }
void orc_shade_query(const OrcScene *sc, const OrcConfig *cfg, uint32_t n, const uint32_t *inst, const uint32_t *prim, const float *uv2, const float *dir3,
                     const float *org3, const float *pay_pdf, const uint32_t *rng, const float *L3, float *out) {
    for (uint32_t i = 0; i < n; i++) {
        float *o = out + (size_t)i * ORC_SQ_STRIDE;
        memset(o, 0, ORC_SQ_STRIDE * sizeof(float));
        const v3 rayDir = v3normalize(V3(dir3[3 * i], dir3[3 * i + 1], dir3[3 * i + 2]));
        Rng r = { rng[i] };
        Surface sf; Mat m;
        const int isLight = hit_surface(sc, cfg, inst[i], prim[i], uv2[2 * i], uv2[2 * i + 1], rayDir, &sf, &m);
        put3(o + ORC_SQ_N, sf.Normal); put3(o + ORC_SQ_T, sf.Tangent); put3(o + ORC_SQ_B, sf.Bitangent); put3(o + ORC_SQ_NG, sf.GeometryNormal);
        o[ORC_SQ_INSIDE] = (float)sf.HitFromInside;
        float pm, pd, pg;
        lobe_probs(&m, &pm, &pd, &pg);
        o[ORC_SQ_AX] = m.Ax; o[ORC_SQ_AY] = m.Ay; o[ORC_SQ_ETA] = m.Eta; o[ORC_SQ_PM] = pm; o[ORC_SQ_PD] = pd; o[ORC_SQ_PG] = pg;
        put3(o + ORC_SQ_BASECOLOR, m.BaseColor); o[ORC_SQ_ROUGHNESS] = m.Roughness;
        put3(o + ORC_SQ_POS, sf.WorldPos);
        put3(o + ORC_SQ_EMITTED, hit_emission(sc, cfg, inst[i], &sf, &m, isLight, 1u, V3(org3[3 * i], org3[3 * i + 1], org3[3 * i + 2]), pay_pdf[i]));
        const v3 V = surf_world_to_tangent(&sf, v3normalize(v3neg(rayDir)));
        if (cfg->EnableSkyMIS) {                                                /* :125-147 */
            v3 w; v4 lv;
            const v3 t = hit_sky_draw(sc, cfg, &sf, &r, &w, &lv);
            put3(o + ORC_SQ_SKY_L, t); put3(o + ORC_SQ_SKY_W, w); put3(o + ORC_SQ_SKY_LV, V3(lv.x, lv.y, lv.z)); o[ORC_SQ_SKY_LV + 3] = lv.w;
            if (lv.w > 0.0f) {
                const Eval e = eval_bsdf(&m, sc, cfg, V, t);
                put_eval(o + ORC_SQ_SKY_EVAL, e);
                if (e.PDF > 0.0f) put3(o + ORC_SQ_SKY_C, nee_term(e, v3s(1.0f), lv));
            }
        }
        put_bits(o + ORC_SQ_LIGHT_GID, 0xFFFFFFFFu);
        if (cfg->EnableMeshMIS && !isLight) {                                   /* :154-184 */
            v3 w; v4 lv; uint32_t lt, li;
            sample_emissive(sc, &r, sf.WorldPos, &w, &lv, &lt, &li);
            put3(o + ORC_SQ_LIGHT_W, w);
            o[ORC_SQ_LIGHT_LV] = lv.x; o[ORC_SQ_LIGHT_LV + 1] = lv.y; o[ORC_SQ_LIGHT_LV + 2] = lv.z; o[ORC_SQ_LIGHT_LV + 3] = lv.w;
            if (li != 0xFFFFFFFFu) put_bits(o + ORC_SQ_LIGHT_GID, sc->xf[li].tri_base + lt);
            if (lv.w > 0.0f) {
                const v3 t = surf_world_to_tangent(&sf, w);
                put3(o + ORC_SQ_LIGHT_L, t);
                const Eval e = eval_bsdf(&m, sc, cfg, V, t);
                put_eval(o + ORC_SQ_LIGHT_EVAL, e);
                if (e.PDF > 0.0f) put3(o + ORC_SQ_LIGHT_C, nee_term(e, v3s(1.0f), lv));
            }
        }
        v3 V2, H;
        BSample ss = hit_sample_bsdf(sc, cfg, &sf, &m, &r, rayDir, &V2, &H);
        put3(o + ORC_SQ_V, V2); put3(o + ORC_SQ_H, H);
        put3(o + ORC_SQ_BSDF_L, ss.L); o[ORC_SQ_BSDF_EVAL] = ss.BxDF.x; o[ORC_SQ_BSDF_EVAL + 1] = ss.BxDF.y; o[ORC_SQ_BSDF_EVAL + 2] = ss.BxDF.z; o[ORC_SQ_BSDF_EVAL + 3] = ss.PDF;
        o[ORC_SQ_VALID] = (ss.L.x != 0.0f || ss.L.y != 0.0f || ss.L.z != 0.0f) ? 1.0f : 0.0f;
        const int wasRefracted = ss.L.z < 0.0f;                                 /* :220-238 */
        const v3 scatterW = surf_tangent_to_world(&sf, ss.L);
        const int rejected = !wasRefracted && v3dot(scatterW, sf.GeometryNormal) < 0.0f;
        if (rejected) { ss.PDF = 0.0f; ss.BxDF = V3(0, 0, 0); }
        put3(o + ORC_SQ_SCATTER, scatterW); put_eval(o + ORC_SQ_SAMPLE, (Eval){ ss.BxDF, ss.PDF });
        o[ORC_SQ_REFRACTED] = (float)wasRefracted; o[ORC_SQ_ENTERED] = (float)(wasRefracted && !sf.HitFromInside); o[ORC_SQ_REJECTED] = (float)rejected;
        if (L3) {
            const v3 t = surf_world_to_tangent(&sf, V3(L3[3 * i], L3[3 * i + 1], L3[3 * i + 2]));
            put3(o + ORC_SQ_USER_L, t); put_eval(o + ORC_SQ_USER_EVAL, eval_bsdf(&m, sc, cfg, V, t));
        }
        put_bits(o + ORC_SQ_RNG, r.seed);
    }
}

/* Miss: SH/Miss.slang:8-76.  miss_emission is what miss_shader and orc_miss_query share: the emitted radiance of a miss along dir at Depth
 * `depth` with BSDF pdf `pdf`, and in .w the sky sampler's pdf of the lookup (1 where none is made). */
static v4 miss_emission(const OrcScene *sc, const OrcConfig *cfg, v3 dir, uint32_t depth, float pdf) {
    v4 c;
    if (cfg->EnableAtmosphere) { v4 z = { 0, 0, 0, 1 }; return z; }            /* :11-14: the sky is the in-scattered sun light, a miss emits nothing */
    if (cfg->ShowEnvMapDirectly || depth > 0) {
        float az = cfg->SkyRotationAzimuth / 180.0f * ORC_PI, al = cfg->SkyRotationAltitude / 180.0f * ORC_PI;
        v3 r = orc_rotate(dir, V3(1, 0, 0), -al);
        r = orc_rotate(r, V3(0, 1, 0), -az);
        float u, v; direction_to_uv(r, &u, &v);
        c = env_sample(sc, u, v);
    } else { v4 z = { 0, 0, 0, 1 }; c = z; }
    v3 e = V3(c.x * cfg->EnvironmentIntensity, c.y * cfg->EnvironmentIntensity, c.z * cfg->EnvironmentIntensity);
    if (cfg->FurnaceTestMode) e = v3s(1.0f);
    if (cfg->EnableSkyMIS && depth > 0) e = v3scale(e, power_heuristic(pdf, c.w));
    v4 r = { e.x, e.y, e.z, c.w };
    return r;
}
static void miss_shader(const OrcScene *sc, const OrcConfig *cfg, Payload *pl) {
    if (!cfg->EnableAtmosphere) {
        const v4 e = miss_emission(sc, cfg, pl->Direction, pl->Depth, pl->PDF);
        pl->Emitted = V3(e.x, e.y, e.z);
    }
    pl->Depth = ORC_MAX_DEPTH;
}
void orc_miss_query(const OrcScene *sc, const OrcConfig *cfg, uint32_t n, const float *dir3, const uint32_t *depth, const float *pay_pdf, float *out) {
    for (uint32_t i = 0; i < n; i++) {
        const v4 e = miss_emission(sc, cfg, V3(dir3[3 * i], dir3[3 * i + 1], dir3[3 * i + 2]), depth[i], pay_pdf[i]);
        float *o = out + (size_t)i * ORC_MQ_STRIDE;
        o[ORC_MQ_RGB] = e.x; o[ORC_MQ_RGB + 1] = e.y; o[ORC_MQ_RGB + 2] = e.z; o[ORC_MQ_PDF] = e.w;
    }
}

/* ------------------------------------------------------------------------------------------------
 * RayGen: SH/RayGen.slang:9-160  (ScatteredInVolume with VolumesCount==0 returns false, :162-263, Q5)
 * ---------------------------------------------------------------------------------------------- */
/* One segment of the path loop (:66-113): trace, shade, clamp (Q3), throughput, Russian roulette (Q4).  Returns 0 when the path ends in the
 * segment (below the planet, or the roulette), 1 otherwise; the loop condition Depth < MaxDepth is the caller's.  hit (optional): the
 * segment's closest hit (hit = 0 on a miss or a volume event). */
static int path_segment(const OrcScene *sc, const OrcConfig *cfg, Payload *pl, v3 *throughput, v3 *pathLight, OrcCounters *cnt, Hit *hit) {
    v3 ro = pl->Origin, rd = v3normalize(pl->Direction);
    pl->Emitted = v3s(0.0f);
    if (hit) memset(hit, 0, sizeof *hit);
    if (cfg->EnableAtmosphere && atm_height(cfg, pl->Origin) < 0.0f) return 0;  /* :76-84: below the surface of the planet */
    cnt->segments++;
    if (!((cfg->VolumesCount || cfg->EnableAtmosphere) && scattered_in_volume(sc, cfg, pl, cnt))) {         /* :86-90 */
        Hit h = trace_bvh(sc, ro, rd, 0.01f, 100000.0f);
        if (hit) *hit = h;
        if (h.hit) closest_hit(sc, cfg, pl, rd, &h, cnt);
        else { miss_shader(sc, cfg, pl); cnt->misses++; }
    }
    v3 contribution = v3mul(pl->Emitted, *throughput);
    if (pl->Depth != 1) {                                                       /* Q3 */
        float lum = v3dot(contribution, V3(0.212671f, 0.715160f, 0.072169f));
        float scale = cfg->MaxLuminance / fmaxf(lum, cfg->MaxLuminance);
        contribution = v3scale(contribution, scale);
    }
    *pathLight = v3add(*pathLight, contribution);
    *throughput = v3mul(*throughput, v3divs(pl->BxDF, pl->PDF));
    float p = fmaxf(throughput->x, fmaxf(throughput->y, throughput->z));
    p = fminf(p, 1.0f);
    if (p < rng_f(&pl->Sampler)) return 0;                                      /* Q4 */
    *throughput = v3divs(*throughput, p);
    return 1;
}

/* :116-128: a finished sample's light is added to acc unless a component is NaN or Inf; a ray split by an atmosphere event carries one channel */
static void fold_sample(v3 *acc, v3 l, int channel) {
    if (isinf(l.x) || isinf(l.y) || isinf(l.z) || isnan(l.x) || isnan(l.y) || isnan(l.z)) return;
    if (channel == -1) *acc = v3add(*acc, l);
    else if (channel == 0) acc->x += l.x; else if (channel == 1) acc->y += l.y; else acc->z += l.z;
}

static v3 trace_one_sample(const OrcScene *sc, const OrcConfig *cfg, Payload *pl, uint32_t W, uint32_t H,
                           uint32_t px, uint32_t py, OrcCounters *cnt) {
    const float *VI = cfg->ViewInverse, *PI = cfg->ProjectionInverse;
    float jx = rng_f(&pl->Sampler) * (0.5f - -0.5f) + -0.5f;                    /* :35 UniformFloat2(-0.5,0.5) */
    float jy = rng_f(&pl->Sampler) * (0.5f - -0.5f) + -0.5f;
    float pcx = (float)px + 0.5f + jx, pcy = (float)py + 0.5f + jy;
    float uvx = pcx / (float)W, uvy = pcy / (float)H;
    float dx = uvx * 2.0f - 1.0f, dy = uvy * 2.0f - 1.0f;
    v3 origin = V3(VI[0] * 0.0f + VI[4] * 0.0f + VI[8] * 0.0f + VI[12] * 1.0f,
                   VI[1] * 0.0f + VI[5] * 0.0f + VI[9] * 0.0f + VI[13] * 1.0f,
                   VI[2] * 0.0f + VI[6] * 0.0f + VI[10] * 0.0f + VI[14] * 1.0f);
    v3 target = V3(PI[0] * dx + PI[4] * dy + PI[8] * 1.0f + PI[12] * 1.0f,
                   PI[1] * dx + PI[5] * dy + PI[9] * 1.0f + PI[13] * 1.0f,
                   PI[2] * dx + PI[6] * dy + PI[10] * 1.0f + PI[14] * 1.0f);
    v3 direction = mat4_dir(VI, v3normalize(target));
    v3 focus = v3add(origin, v3scale(direction, fmaxf(cfg->FocusDistance, 0.001f)));
    float cx, cy; rng_circle(&pl->Sampler, &cx, &cy);
    float ox = cx * 0.5f * cfg->DepthOfFieldStrength, oy = cy * 0.5f * cfg->DepthOfFieldStrength;
    v3 right = V3(VI[0], VI[1], VI[2]);     /* M[0][0],M[1][0],M[2][0] = column 0 */
    v3 upv = V3(VI[4], VI[5], VI[6]);       /* column 1 */
    origin = v3add(origin, v3add(v3scale(right, ox), v3scale(upv, oy)));
    direction = v3normalize(v3sub(focus, origin));

    pl->Depth = 0; pl->Origin = origin; pl->Direction = direction;
    pl->BxDF = v3s(1.0f); pl->PDF = 1.0f; pl->Emitted = v3s(0.0f); pl->InMedium = 0; pl->VolumeDepth = 0; pl->ColorChannel = -1;
    v3 throughput = v3s(1.0f), pathLight = v3s(0.0f);
    cnt->paths++;
    while (pl->Depth < cfg->MaxDepth && path_segment(sc, cfg, pl, &throughput, &pathLight, cnt, NULL)) {}
    return pathLight;
}

void orc_bounce_query(const OrcScene *s, const OrcConfig *cfg, uint32_t n, const float *in, uint32_t flags, float *out, uint32_t *survivors) {
    uint32_t alive_n = 0;
    memset(out, 0, (size_t)n * ORC_BQ_OUT_STRIDE * sizeof(float));
    for (uint32_t i = 0; i < n; i++) {
        const float *r = in + (size_t)i * ORC_BQ_IN_STRIDE;
        float *o = out + (size_t)i * ORC_BQ_OUT_STRIDE;
        uint32_t dflags, seed; memcpy(&dflags, r + ORC_BQ_IN_DFLAGS, 4); memcpy(&seed, r + ORC_BQ_IN_RNG, 4);
        Payload pl; memset(&pl, 0, sizeof(pl));
        pl.Origin = V3(r[ORC_BQ_IN_ORG], r[ORC_BQ_IN_ORG + 1], r[ORC_BQ_IN_ORG + 2]); pl.PDF = r[ORC_BQ_IN_PDF];
        pl.Direction = V3(r[ORC_BQ_IN_DIR], r[ORC_BQ_IN_DIR + 1], r[ORC_BQ_IN_DIR + 2]); pl.Sampler.seed = seed;
        pl.Depth = dflags & 0x07FFFFFFu; pl.ColorChannel = (int)((dflags >> 27) & 3u) - 1; pl.InMedium = (int)(dflags >> 31);
        pl.MediumColor = V3(r[ORC_BQ_IN_MEDIUM], r[ORC_BQ_IN_MEDIUM + 1], r[ORC_BQ_IN_MEDIUM + 2]);
        pl.MediumDensity = r[ORC_BQ_IN_MEDIUM + 3]; pl.MediumAnisotropy = r[ORC_BQ_IN_MEDIUM_G];
        v3 throughput = V3(r[ORC_BQ_IN_THR], r[ORC_BQ_IN_THR + 1], r[ORC_BQ_IN_THR + 2]);
        v3 pathLight = V3(r[ORC_BQ_IN_RAD], r[ORC_BQ_IN_RAD + 1], r[ORC_BQ_IN_RAD + 2]);
        OrcCounters c; memset(&c, 0, sizeof(c));
        Hit h;
        const int alive = path_segment(s, cfg, &pl, &throughput, &pathLight, &c, &h) && pl.Depth < cfg->MaxDepth;
        uint32_t inst = 0xFFFFFFFFu, prim = 0xFFFFFFFFu;
        if (h.hit) { inst = s->tris[h.tri].inst; prim = s->tris[h.tri].prim; o[ORC_BQ_OUT_T] = h.t; o[ORC_BQ_OUT_U] = h.u; o[ORC_BQ_OUT_V] = h.v; }
        memcpy(o + ORC_BQ_OUT_INST, &inst, 4); memcpy(o + ORC_BQ_OUT_PRIM, &prim, 4);
        o[ORC_BQ_OUT_ALIVE] = alive ? 1.0f : 0.0f;
        memcpy(o + ORC_BQ_OUT_SAMPLE, r + ORC_BQ_IN_SAMPLE, 16);
        if (alive) {
            float *x = o + ORC_BQ_OUT_NEXT;
            const uint32_t nd = pl.Depth | ((uint32_t)(pl.ColorChannel + 1) << 27) | (pl.InMedium ? 0x80000000u : 0u);
            x[ORC_BQ_IN_ORG] = pl.Origin.x; x[ORC_BQ_IN_ORG + 1] = pl.Origin.y; x[ORC_BQ_IN_ORG + 2] = pl.Origin.z; x[ORC_BQ_IN_PDF] = pl.PDF;
            x[ORC_BQ_IN_DIR] = pl.Direction.x; x[ORC_BQ_IN_DIR + 1] = pl.Direction.y; x[ORC_BQ_IN_DIR + 2] = pl.Direction.z;
            memcpy(x + ORC_BQ_IN_RNG, &pl.Sampler.seed, 4);
            x[ORC_BQ_IN_THR] = throughput.x; x[ORC_BQ_IN_THR + 1] = throughput.y; x[ORC_BQ_IN_THR + 2] = throughput.z; memcpy(x + ORC_BQ_IN_DFLAGS, &nd, 4);
            x[ORC_BQ_IN_RAD] = pathLight.x; x[ORC_BQ_IN_RAD + 1] = pathLight.y; x[ORC_BQ_IN_RAD + 2] = pathLight.z; memcpy(x + ORC_BQ_IN_SLOT, &i, 4);
            if (pl.InMedium) {
                x[ORC_BQ_IN_MEDIUM] = pl.MediumColor.x; x[ORC_BQ_IN_MEDIUM + 1] = pl.MediumColor.y; x[ORC_BQ_IN_MEDIUM + 2] = pl.MediumColor.z;
                x[ORC_BQ_IN_MEDIUM + 3] = pl.MediumDensity; x[ORC_BQ_IN_MEDIUM_G] = pl.MediumAnisotropy;
            }
            alive_n++;
        } else {
            float *acc4 = o + ORC_BQ_OUT_SAMPLE;
            if (flags & ORC_BQ_STORE) memset(acc4, 0, 16);
            v3 acc = V3(acc4[0], acc4[1], acc4[2]);
            fold_sample(&acc, pathLight, pl.ColorChannel);
            acc4[0] = acc.x; acc4[1] = acc.y; acc4[2] = acc.z;
            if (flags & ORC_BQ_CARRY) memcpy(o + ORC_BQ_OUT_CARRY, &pl.Sampler.seed, 4);
        }
    }
    *survivors = alive_n;
}

void orc_sample_pixel(const OrcScene *s, const OrcConfig *cfg, uint32_t W, uint32_t H,
                      uint32_t x, uint32_t y, uint32_t seed, float out_rgb[3], uint32_t *segments_out) {
    Payload pl; memset(&pl, 0, sizeof(pl));
    pl.Sampler.seed = y + W * x + seed;                                         /* :28 (Q13) */
    OrcCounters c; memset(&c, 0, sizeof(c));
    v3 l = trace_one_sample(s, cfg, &pl, W, H, x, y, &c);
    if (pl.ColorChannel == 0) { l.y = 0.0f; l.z = 0.0f; } else if (pl.ColorChannel == 1) { l.x = 0.0f; l.z = 0.0f; } else if (pl.ColorChannel == 2) { l.x = 0.0f; l.y = 0.0f; }
    out_rgb[0] = l.x; out_rgb[1] = l.y; out_rgb[2] = l.z;
    if (segments_out) *segments_out = (uint32_t)c.segments;
}

typedef struct {
    const OrcScene *s; const OrcConfig *cfg; uint32_t W, H, frameCount, seed, chunk, rank, world, band;
    float *image; int tid, nthreads; OrcCounters cnt;
} RenderJob;

static void *render_thread(void *arg) {
    RenderJob *j = (RenderJob *)arg;
    const OrcConfig *cfg = j->cfg;
    uint32_t S = cfg->ScreenSplitCount ? cfg->ScreenSplitCount : 1;
    uint32_t LW = (j->W + S - 1) / S, LH = (j->H + S - 1) / S;                  /* PT/PathTracer.cpp:146-150 */
    for (uint32_t ly = (uint32_t)j->tid; ly < LH; ly += (uint32_t)j->nthreads) {
        for (uint32_t lx = 0; lx < LW; lx++) {
            uint32_t x = lx * S + j->chunk % S, y = ly * S + j->chunk / S;      /* SH/RayGen.slang:17-22 */
            if (x >= j->W || y >= j->H) continue;
            if (((y / j->band) % j->world) != j->rank) continue;                /* image-tile partition */
            Payload pl; memset(&pl, 0, sizeof(pl));
            pl.Sampler.seed = y + j->W * x + j->seed;                           /* :28 */
            float *px = j->image + ((size_t)y * j->W + x) * 4;
            v3 prev = V3(px[0], px[1], px[2]);
            v3 acc = v3s(0.0f);
            for (uint32_t i = 0; i < cfg->SampleCount; i++) {
                v3 l = trace_one_sample(j->s, cfg, &pl, j->W, j->H, x, y, &j->cnt);
                fold_sample(&acc, l, pl.ColorChannel);
            }
            acc = v3divs(acc, (float)cfg->SampleCount);
            v3 color;
            if (j->frameCount > 0) { float a = 1.0f / (float)(j->frameCount + 1); color = v3lerp(prev, acc, a); }  /* :132-141 */
            else color = acc;
            if (j->frameCount == 0 && j->chunk == 0) {                          /* :144-157 */
                for (uint32_t a = 0; a < S; a++) for (uint32_t b = 0; b < S; b++) {
                    uint32_t qx = x + a, qy = y + b;
                    if (qx < j->W && qy < j->H) { float *q = j->image + ((size_t)qy * j->W + qx) * 4; q[0] = color.x; q[1] = color.y; q[2] = color.z; q[3] = 1.0f; }
                }
            }
            px[0] = color.x; px[1] = color.y; px[2] = color.z; px[3] = 1.0f;
        }
    }
    return NULL;
}

void orc_render(const OrcScene *s, const OrcConfig *cfg, uint32_t W, uint32_t H,
                uint32_t frame0, uint32_t nframes, uint32_t base_seed,
                uint32_t rank, uint32_t world, uint32_t band_rows,
                float *image, int nthreads, OrcCounters *counters) {
    if (nthreads <= 0) { long n = sysconf(_SC_NPROCESSORS_ONLN); nthreads = n > 0 ? (int)n : 1; }
    if (nthreads > 256) nthreads = 256;
    if (world == 0) world = 1;
    if (band_rows == 0) band_rows = 1;
    uint32_t S = cfg->ScreenSplitCount ? cfg->ScreenSplitCount : 1;
    OrcCounters total; memset(&total, 0, sizeof(total));
    /* PT/PathTracer.cpp:122-156: dispatch d renders chunk d % S^2 with FrameCount = floor(d / S^2) */
    for (uint32_t f = frame0; f < frame0 + nframes; f++) {
        for (uint32_t chunk = 0; chunk < S * S; chunk++) {
            uint32_t dispatch = f * S * S + chunk;
            uint32_t seed = orc_pcg_hash(base_seed + dispatch);
            pthread_t th[256]; RenderJob jobs[256];
            for (int t = 0; t < nthreads; t++) {
                RenderJob *j = &jobs[t];
                j->s = s; j->cfg = cfg; j->W = W; j->H = H; j->frameCount = f; j->seed = seed; j->chunk = chunk;
                j->rank = rank; j->world = world; j->band = band_rows; j->image = image; j->tid = t; j->nthreads = nthreads;
                memset(&j->cnt, 0, sizeof(j->cnt));
                pthread_create(&th[t], NULL, render_thread, j);
            }
            for (int t = 0; t < nthreads; t++) {
                pthread_join(th[t], NULL);
                total.paths += jobs[t].cnt.paths; total.segments += jobs[t].cnt.segments; total.surface_hits += jobs[t].cnt.surface_hits;
                total.misses += jobs[t].cnt.misses; total.shadow_rays += jobs[t].cnt.shadow_rays; total.medium_events += jobs[t].cnt.medium_events;
            }
        }
    }
    if (counters) *counters = total;
}

/* ------------------------------------------------------------------------------------------------
 * Host one-offs
 * ---------------------------------------------------------------------------------------------- */
void orc_default_config(OrcConfig *c) {                                         /* PT/PathTracer.h:197-233 */
    memset(c, 0, sizeof(*c));
    for (int i = 0; i < 4; i++) c->ViewInverse[i * 5] = c->ProjectionInverse[i * 5] = 1.0f;
    c->SampleCount = 1; c->MaxDepth = 200; c->MaxLuminance = 500.0f; c->FocusDistance = 1.0f; c->DepthOfFieldStrength = 0.0f;
    c->SkyRotationAzimuth = 0.0f; c->SkyRotationAltitude = 0.0f; c->EnvironmentIntensity = 1.0f;
    c->EmissiveMeshSamplingPDFBias = 0.0f; c->ScreenSplitCount = 1;
    c->EnableSkyMIS = 1; c->EnableMeshMIS = 1; c->ShowEnvMapDirectly = 1; c->UseOnlyGeometryNormals = 0;
    c->UseEnergyCompensation = 1; c->FurnaceTestMode = 0;
    /* atmosphere, PT/PathTracer.h:221-232 */
    c->EnableAtmosphere = 0; c->PlanetPosition[0] = 0.0f; c->PlanetPosition[1] = 6360e3f + 1000.0f; c->PlanetPosition[2] = 0.0f;
    c->PlanetRadius = 6360e3f; c->AtmosphereHeight = 100e3f;
    for (int k = 0; k < 3; k++) { c->RayleighScatteringCoefficientMultiplier[k] = 1.0f; c->MieScatteringCoefficientMultiplier[k] = 1.0f; c->OzoneAbsorptionCoefficientMultiplier[k] = 1.0f; }
    c->RayleighDensityFalloff = 8000.0f; c->MieDensityFalloff = 1200.0f; c->OzoneDensityFalloff = 5000.0f; c->OzonePeak = 22000.0f;
    c->SunColor[0] = 1.0f; c->SunColor[1] = 0.956f; c->SunColor[2] = 0.88f;
}

/* PT/PathTracer.cpp:1137-1332 (Q1 kept: lowEnergyCounter++ before the store) */
float orc_build_env_alias(float *pixels, uint32_t width, uint32_t height, OrcAliasEntry *aliasMap) {
    const uint32_t size = width * height;
    float *importance = (float *)malloc(sizeof(float) * (size_t)size);
    float cosTheta0 = 1.0f;
    const float stepPhi = (float)2.0f * (float)3.14159265358979323846 / (float)width;
    const float stepTheta = (float)3.14159265358979323846 / (float)height;
    for (uint32_t y = 0; y < height; ++y) {
        const float theta1 = (float)(y + 1) * stepTheta;
        const float cosTheta1 = cosf(theta1);
        const float area = (cosTheta0 - cosTheta1) * stepPhi;
        cosTheta0 = cosTheta1;
        for (uint32_t x = 0; x < width; ++x) {
            const uint32_t idx = y * width + x, idx4 = idx * 4;
            importance[idx] = area * fmaxf(pixels[idx4], fmaxf(pixels[idx4 + 1], pixels[idx4 + 2]));
        }
    }
    float sum = 0.0f;                                      /* std::accumulate(..., 0.0f): sequential fp32 */
    for (uint32_t i = 0; i < size; i++) sum = sum + importance[i];
    float average = sum / (float)size;
    for (uint32_t i = 0; i < size; i++) {
        aliasMap[i].Importance = (average == 0.0f) ? 0.0f : importance[i] / average;
        aliasMap[i].Alias = i;
    }
    uint32_t *partition = (uint32_t *)calloc((size_t)size + 1, sizeof(uint32_t));  /* +1: the reference writes [size] when every texel is low (UB there) */
    uint32_t low = 0u, high = size;
    for (uint32_t i = 0; i < size; ++i) {
        if (aliasMap[i].Importance < 1.0f) { low++; partition[low] = i; }
        else { high--; partition[high] = i; }
    }
    for (low = 0; low < high && high < size; low++) {
        const uint32_t li = partition[low], hi = partition[high];
        aliasMap[li].Alias = hi;
        const float diff = 1.0f - aliasMap[li].Importance;
        aliasMap[hi].Importance -= diff;
        if (aliasMap[hi].Importance < 1.0f) high++;
    }
    for (uint32_t i = 0; i < size; ++i) {
        const uint32_t idx4 = i * 4;
        pixels[idx4 + 3] = (sum == 0.0f) ? 0.0f : fmaxf(pixels[idx4], fmaxf(pixels[idx4 + 1], pixels[idx4 + 2])) / sum;
    }
    free(partition); free(importance);
    return sum;
}

/* PT/Editor.cpp:45-48,1042-1051 -> PT/FlyCamera.cpp:110-140 (InitializeFromMatrices), :96-108, :84-94.
 * view = CameraAsset::ViewMatrix (column-major).  Q2: yfov ignored (45 deg), roll dropped. */
static void mat4_inverse_rigidish(const float m[16], float out[16]) {
    /* general 4x4 inverse by cofactors in double */
    double a[16], inv[16];
    for (int i = 0; i < 16; i++) a[i] = m[i];
    inv[0] = a[5] * a[10] * a[15] - a[5] * a[11] * a[14] - a[9] * a[6] * a[15] + a[9] * a[7] * a[14] + a[13] * a[6] * a[11] - a[13] * a[7] * a[10];
    inv[4] = -a[4] * a[10] * a[15] + a[4] * a[11] * a[14] + a[8] * a[6] * a[15] - a[8] * a[7] * a[14] - a[12] * a[6] * a[11] + a[12] * a[7] * a[10];
    inv[8] = a[4] * a[9] * a[15] - a[4] * a[11] * a[13] - a[8] * a[5] * a[15] + a[8] * a[7] * a[13] + a[12] * a[5] * a[11] - a[12] * a[7] * a[9];
    inv[12] = -a[4] * a[9] * a[14] + a[4] * a[10] * a[13] + a[8] * a[5] * a[14] - a[8] * a[6] * a[13] - a[12] * a[5] * a[10] + a[12] * a[6] * a[9];
    inv[1] = -a[1] * a[10] * a[15] + a[1] * a[11] * a[14] + a[9] * a[2] * a[15] - a[9] * a[3] * a[14] - a[13] * a[2] * a[11] + a[13] * a[3] * a[10];
    inv[5] = a[0] * a[10] * a[15] - a[0] * a[11] * a[14] - a[8] * a[2] * a[15] + a[8] * a[3] * a[14] + a[12] * a[2] * a[11] - a[12] * a[3] * a[10];
    inv[9] = -a[0] * a[9] * a[15] + a[0] * a[11] * a[13] + a[8] * a[1] * a[15] - a[8] * a[3] * a[13] - a[12] * a[1] * a[11] + a[12] * a[3] * a[9];
    inv[13] = a[0] * a[9] * a[14] - a[0] * a[10] * a[13] - a[8] * a[1] * a[14] + a[8] * a[2] * a[13] + a[12] * a[1] * a[10] - a[12] * a[2] * a[9];
    inv[2] = a[1] * a[6] * a[15] - a[1] * a[7] * a[14] - a[5] * a[2] * a[15] + a[5] * a[3] * a[14] + a[13] * a[2] * a[7] - a[13] * a[3] * a[6];
    inv[6] = -a[0] * a[6] * a[15] + a[0] * a[7] * a[14] + a[4] * a[2] * a[15] - a[4] * a[3] * a[14] - a[12] * a[2] * a[7] + a[12] * a[3] * a[6];
    inv[10] = a[0] * a[5] * a[15] - a[0] * a[7] * a[13] - a[4] * a[1] * a[15] + a[4] * a[3] * a[13] + a[12] * a[1] * a[7] - a[12] * a[3] * a[5];
    inv[14] = -a[0] * a[5] * a[14] + a[0] * a[6] * a[13] + a[4] * a[1] * a[14] - a[4] * a[2] * a[13] - a[12] * a[1] * a[6] + a[12] * a[2] * a[5];
    inv[3] = -a[1] * a[6] * a[11] + a[1] * a[7] * a[10] + a[5] * a[2] * a[11] - a[5] * a[3] * a[10] - a[9] * a[2] * a[7] + a[9] * a[3] * a[6];
    inv[7] = a[0] * a[6] * a[11] - a[0] * a[7] * a[10] - a[4] * a[2] * a[11] + a[4] * a[3] * a[10] + a[8] * a[2] * a[7] - a[8] * a[3] * a[6];
    inv[11] = -a[0] * a[5] * a[11] + a[0] * a[7] * a[9] + a[4] * a[1] * a[11] - a[4] * a[3] * a[9] - a[8] * a[1] * a[7] + a[8] * a[3] * a[5];
    inv[15] = a[0] * a[5] * a[10] - a[0] * a[6] * a[9] - a[4] * a[1] * a[10] + a[4] * a[2] * a[9] + a[8] * a[1] * a[6] - a[8] * a[2] * a[5];
    double det = a[0] * inv[0] + a[1] * inv[4] + a[2] * inv[8] + a[3] * inv[12];
    det = 1.0 / det;
    for (int i = 0; i < 16; i++) out[i] = (float)(inv[i] * det);
}

void orc_camera_from_view(const float view[16], float aspect, float viewInv_out[16], float projInv_out[16]) {
    float invView[16];
    mat4_inverse_rigidish(view, invView);
    v3 pos = V3(invView[12], invView[13], invView[14]);
    /* forward = -(view[0][2], view[1][2], view[2][2]) (glm column-major: view[c][r]) */
    v3 fwd = v3normalize(v3neg(V3(view[0 * 4 + 2], view[1 * 4 + 2], view[2 * 4 + 2])));
    const float RAD2DEG = 57.295779513082320876798154814105f, DEG2RAD = 0.01745329251994329576923690768489f;
    float yaw = atan2f(fwd.z, fwd.x) * RAD2DEG;
    float pitch = asinf(fwd.y) * RAD2DEG;
    /* PT/PathTracer.cpp:578: projection perspective(radians(45), aspect, 0.1, 100); FlyCamera re-derives fov/aspect */
    float tanHalf0 = tanf((45.0f * DEG2RAD) / 2.0f);
    float P00 = 1.0f / (aspect * tanHalf0), P11 = 1.0f / tanHalf0;
    float fov = (2.0f * atanf(1.0f / P11)) * RAD2DEG;
    float asp = P11 / P00;
    /* UpdateCameraVectors :96-108 */
    v3 front = v3normalize(V3(cosf(yaw * DEG2RAD) * cosf(pitch * DEG2RAD), sinf(pitch * DEG2RAD), sinf(yaw * DEG2RAD) * cosf(pitch * DEG2RAD)));
    v3 right = v3normalize(v3cross(front, V3(0, 1, 0)));
    v3 up = v3normalize(v3cross(right, front));
    /* glm::lookAt RH (:84-88): f = normalize(center-eye); s = normalize(cross(f, up)); u = cross(s, f) */
    v3 f = v3normalize(v3sub(v3add(pos, front), pos));
    v3 s = v3normalize(v3cross(f, up));
    v3 u = v3cross(s, f);
    /* inverse(view) for an orthonormal basis: columns s, u, -f, pos */
    float vi[16] = { s.x, s.y, s.z, 0.0f, u.x, u.y, u.z, 0.0f, -f.x, -f.y, -f.z, 0.0f, pos.x, pos.y, pos.z, 1.0f };
    memcpy(viewInv_out, vi, sizeof(vi));
    /* glm::perspective RH_ZO(radians(fov), asp, 0.1, 1000) (:90-94) and its analytic inverse */
    float tanHalf = tanf((fov * DEG2RAD) / 2.0f);
    float n = 0.1f, fz = 1000.0f;
    float A = 1.0f / (asp * tanHalf), B = 1.0f / tanHalf, C = fz / (n - fz), D = -(fz * n) / (fz - n);
    float pi_[16] = { 1.0f / A, 0, 0, 0, 0, 1.0f / B, 0, 0, 0, 0, 0, 1.0f / D, 0, 0, -1.0f, C / D };
    memcpy(projInv_out, pi_, sizeof(pi_));
}

/* ------------------------------------------------------------------------------------------------
 * AddDensityDataToVolume after the OpenVDB file read: PT/PathTracer.cpp:1391-1452
 * ---------------------------------------------------------------------------------------------- */
void orc_prepare_density_grid(const int32_t indexMin[3], const uint32_t dim[3], float *values, const float *temperature, float temperatureMin, float temperatureMax,
                              float *maxDensities32, float cornerMin[3], float cornerMax[3], float *maxDensityInTheGrid) {
    const size_t n = (size_t)dim[0] * dim[1] * dim[2];
    float maxDensity = values[0];                                               /* tools::minMax(tree, true).max(), :1393 */
    for (size_t i = 1; i < n; i++) if (values[i] > maxDensity) maxDensity = values[i];
    *maxDensityInTheGrid = maxDensity;
    float maxDim = 0.0f;                                                        /* :1411-1420: the AABB is the index bbox scaled into about [-1, 1] */
    for (int k = 0; k < 3; k++) {
        const int lo = indexMin[k], hi = indexMin[k] + (int)dim[k] - 1;
        cornerMin[k] = (float)lo; cornerMax[k] = (float)hi;
        const float m = fmaxf(fabsf((float)lo), fabsf((float)hi));
        if (m > maxDim) maxDim = m;
    }
    for (int k = 0; k < 3; k++) { cornerMin[k] /= maxDim; cornerMax[k] /= maxDim; }
    for (int i = 0; i < 32768; i++) maxDensities32[i] = 0.0f;
    const int dx = (int)dim[0], dy = (int)dim[1], dz = (int)dim[2];
    for (int z = 0; z < dz; z++)
        for (int y = 0; y < dy; y++)
            for (int x = 0; x < dx; x++) {
                const size_t at = ((size_t)z * dy + (size_t)(dy - 1 - y)) * dx + (size_t)x;   /* :1432: Y flipped */
                const float density = orc_clamp(values[at] / maxDensity, 0.0f, 1.0f);
                const int cell = ((x * 32) / dx) + ((y * 32) / dy) * 32 + ((z * 32) / dz) * 1024;
                if (maxDensities32[cell] < density) maxDensities32[cell] = density;
                if (temperature) {                                              /* :1440-1450: the normalised temperature lands in the DENSITY grid */
                    float t = fmaxf((temperature[at] - temperatureMin) / (temperatureMax - temperatureMin), 0.0f);
                    if (t > 0.0f) values[at] = t;
                }
            }
}
float orc_grid_transmittance(const OrcConfig *cfg, uint32_t seed, const float o[3], const float d[3], float rayDepth) {
    Rng r; r.seed = seed;
    return volumes_transmittance(cfg, &r, V3(o[0], o[1], o[2]), V3(d[0], d[1], d[2]), rayDepth);
}
/* both volume walks on caller-supplied rays / seeds (the counterpart of b200pt_volume_walks) */
void orc_volume_walks(const OrcConfig *cfg, uint32_t n, const float *org, const float *dir, const uint32_t *seeds, float rayDepth,
                      float *T, float *scatter, int32_t *vol, uint32_t *rng2) {
    for (uint32_t i = 0; i < n; i++) {
        v3 o = V3(org[3 * i], org[3 * i + 1], org[3 * i + 2]), d = V3(dir[3 * i], dir[3 * i + 1], dir[3 * i + 2]);
        Rng r; r.seed = seeds[i];
        T[i] = volumes_transmittance(cfg, &r, o, d, rayDepth);
        rng2[2 * i] = r.seed;
        r.seed = seeds[i];
        float distances[ORC_MAX_VOLUMES]; int indices[ORC_MAX_VOLUMES];             /* SH/RayGen.slang:164-209 */
        const int nv = (int)(cfg->VolumesCount < ORC_MAX_VOLUMES ? cfg->VolumesCount : ORC_MAX_VOLUMES);
        for (int k = 0; k < nv; k++) { VolIsect is = vol_intersect(o, d, cfg->Volumes[k].CornerMin, cfg->Volumes[k].CornerMax); distances[k] = fmaxf(0.0f, is.Near); indices[k] = k; }
        for (int a = 0; a < nv; a++)
            for (int b = a + 1; b < nv; b++)
                if (distances[b] < distances[a]) { float td = distances[a]; int ti = indices[a]; distances[a] = distances[b]; indices[a] = indices[b]; distances[b] = td; indices[b] = ti; }
        float sd = -1.0f; int sv = -1;
        for (int k = 0; k < nv; k++) {
            float t = vol_scatter_distance(cfg, &cfg->Volumes[indices[k]], o, d, &r, rayDepth, sd);
            if (t >= 0.0f && (t < sd || sd < 0.0f)) { sd = t; sv = indices[k]; }
        }
        scatter[i] = sd; vol[i] = sv; rng2[2 * i + 1] = r.seed;
    }
}
float orc_grid_sample(const OrcConfig *cfg, uint32_t volume, uint32_t seed, const float x[3]) {
    Rng r; r.seed = seed;
    const OrcVolume *v = &cfg->Volumes[volume];
    return grid_sample(v, &cfg->Grids[v->DensityDataIndex], &r, V3(x[0], x[1], x[2]));
}
/* atmosphere KAT hooks: one ratio-tracked transmittance walk, one Rayleigh-phase sample, one sun-disk sample */
float orc_atm_transmittance(const OrcConfig *cfg, uint32_t seed, const float o[3], const float d[3], int channel) {
    Rng r; r.seed = seed;
    v3 T = atm_transmittance(cfg, &r, V3(o[0], o[1], o[2]), V3(d[0], d[1], d[2]), channel);
    return channel == 0 ? T.x : (channel == 1 ? T.y : T.z);
}
void orc_atm_samples(const OrcConfig *cfg, uint32_t seed, const float incident[3], float rayleigh_dir[3], float sun_dir[3], float sun_color_pdf[4]) {
    Rng r; r.seed = seed;
    v3 a = rng_rayleigh(&r, V3(incident[0], incident[1], incident[2]));
    rayleigh_dir[0] = a.x; rayleigh_dir[1] = a.y; rayleigh_dir[2] = a.z;
    v3 s; v4 cp; sample_sun_disk(cfg, &r, &s, &cp);
    sun_dir[0] = s.x; sun_dir[1] = s.y; sun_dir[2] = s.z; sun_color_pdf[0] = cp.x; sun_color_pdf[1] = cp.y; sun_color_pdf[2] = cp.z; sun_color_pdf[3] = cp.w;
}
void orc_blackbody(float kelvin, float out[3]) { v3 c = blackbody(kelvin); out[0] = c.x; out[1] = c.y; out[2] = c.z; }
