/*
 * pt_oracle.h -- CPU ORACLE (TEST INFRASTRUCTURE ONLY).
 *
 * A plain-C restatement of the Monte-Carlo estimator of Zydak/Vulkan-Path-Tracer
 * (reference paths relative to the reference repository):
 *   PathTracer/Shaders/{Defines,Sampler,RTCommon,Surface,Material,ClosestHit,Miss,RayGen,Volume,Atmosphere}.slang
 *   PathTracer/Shaders/PostProcess/{BloomDownSample,BloomUpSample,Tonemap}.slang
 *   PathTracer/PathTracer.cpp:122-156 (dispatch bookkeeping), :1137-1332 (env alias table)
 *   PathTracer/PostProcessor.cpp:128-246, PathTracer/FlyCamera.cpp:84-140
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load this library.  The product (vulkan-path-tracer_b200/) never links or calls it.
 *
 * PARITY PIN STATUS: "parity unpinned" against a Vulkan RENDER.  The reference ships no tests,
 * golden images or fixtures for this path and cannot be built here (SURVEY.md section 8c).
 * What pins the oracle instead:
 *   (a) reference-produced data: the shipped energy-compensation tables Assets/LookupTables/[*].bin were
 *       baked by the reference's own shaders from the hot-path functions GGXSampleAnisotopic /
 *       EvaluateReflection / EvaluateRefraction / DielectricFresnel / UniformFloat; the oracle's restated
 *       baker (orc_bake_*_texel) reproduces them within Monte-Carlo noise (tests/test_oracle_kat.py);
 *   (b) analytic known-answer tests derived from the reference source (furnace mode, PCG sequences,
 *       Fresnel/ACES fixed points, bloom mip sizes, alias-table invariants, LUT ranges, fixture facts).
 * The volume and atmosphere restatements (Volume.slang, Atmosphere.slang, RayGen.slang:162-471, PathTracer.cpp:1346-1528) are pinned by (b) only:
 * the reference ships no .vdb asset and no render with known settings, and the NanoVDB / OpenVDB reads are restated from those libraries'
 * published behaviour (OpenVDB 12.0.1 is absent from the reference tree) -- "parity unpinned" against reference-produced data for that part.
 */
#ifndef PT_ORACLE_H
#define PT_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { float pos[3]; float nrm[3]; float uv[2]; } OrcVertex;       /* SH/Bindings.slang:7-12  (32 B) */

typedef struct {                                                             /* PT/PathTracer.h:12-34  (112 B) */
    float BaseColor[3], EmissiveColor[3], SpecularColor[3], MediumColor[3], MediumEmissiveColor[3];
    float Metallic, Roughness, IOR, Transmission, Anisotropy, AnisotropyRotation;
    float MediumDensity, MediumAnisotropy;
    uint32_t BaseColorTextureIndex, NormalTextureIndex, RoughnessTextureIndex, MetallicTextureIndex, EmissiveTextureIndex;
} OrcMaterial;

typedef struct { uint32_t width, height, channels; uint32_t _pad; const uint8_t *data; } OrcTexture; /* channels 4 (RGBA8) or 1 (R8) */
typedef struct { const OrcVertex *verts; const uint32_t *indices; uint32_t nverts, nindices; } OrcMesh;
typedef struct { float transform[16]; uint32_t mesh, material; } OrcInstance; /* column-major (glm) */
typedef struct { uint32_t Alias; float Importance; } OrcAliasEntry;           /* SH/Bindings.slang:1-5 */

typedef struct {
    const OrcMesh *meshes;         uint32_t nmeshes;   uint32_t _p0;
    const OrcMaterial *materials;  uint32_t nmaterials; uint32_t _p1;
    const OrcTexture *textures;    uint32_t ntextures; uint32_t _p2;
    const OrcInstance *instances;  uint32_t ninstances; uint32_t _p3;
    const float *env_rgba;         /* envW*envH*4, alpha = pdf (orc_build_env_alias) */
    const OrcAliasEntry *env_alias;
    uint32_t envW, envH;
    const float *lut_reflect;      /* 64x64x32   [layer][y][x]  PT/PathTracer.cpp:199 */
    const float *lut_refract_out;  /* 128x128x32               :200 */
    const float *lut_refract_in;   /* 128x128x32               :201 */
} OrcSceneDesc;

/* AABB volume: the fields of VolumeGPU (PT/PathTracer.h:341-395, SH/Volume.slang:20-52).  DensityDataIndex == -1: homogeneous;
 * >= 0: index into OrcConfig::Grids (heterogeneous: the density / temperature data AddDensityDataToVolume prepared, PT/PathTracer.cpp:1346-1516). */
typedef struct {
    float CornerMin[3], CornerMax[3];
    float Color[3], EmissiveColor[3];
    float Density, Anisotropy, Alpha, DropletSize;
    uint32_t ApproximatedScattering;     /* m_ApproximatedScattering: anisotropy / density decay with the depth (SH/Volume.slang:150-166) */
    float ApproximatedScatteringFalloff; /* (0.8) */
    float TemperatureColor[3];           /* (1, 0.5, 0) used when UseBlackbody == 0 */
    int32_t DensityDataIndex;            /* (-1) */
    float MaxDensityInTheGrid;           /* set by orc_prepare_density_grid */
    int32_t UseBlackbody, HasTemperatureData;   /* (1, 0) */
    float TemperatureGamma, TemperatureScale, EmissiveColorGamma;   /* (1, 1, 1) */
    int32_t KelvinMin, KelvinMax;        /* (500, 8000) */
    float GridSharpness;                 /* (1) */
} OrcVolume;

/* Density data of one heterogeneous volume.  The reference keeps it in a NanoVDB buffer built from an OpenVDB FloatGrid (OpenVDB 12.0.1 is a vcpkg
 * dependency, VulkanHelper/vcpkg.json, absent from the reference tree -- and so is PNanoVDB.h, which SH/Volume.slang:6-7 includes).  What the shader
 * reads from it (SH/Volume.slang:69-117) is restated here over a DENSE copy of the same values: pnanovdb_grid_get_world_bbox (the index bbox
 * [min, max + 1] through the grid's map, NanoVDB GridStats), pnanovdb_grid_world_to_indexf (float inverse map), pnanovdb_hdda_pos_to_ijk (floor),
 * pnanovdb_root_get_bbox_min/max (the active-voxel bbox) and a value read at an index coordinate inside that bbox. */
typedef struct {
    const float *Values;          /* [z][y][x] over the active-voxel bbox, x fastest: tree().getValue(IndexMin + (x, y, z)) AFTER the temperature patch of PathTracer.cpp:1437-1450 */
    const float *MaxDensities;    /* 32 x 32 x 32 majorants, PathTracer.cpp:1414-1452 */
    int32_t IndexMin[3];          /* evalActiveVoxelBoundingBox().min() */
    uint32_t Dim[3];              /* evalActiveVoxelDim() */
    double WorldBBox[6];          /* min xyz, max xyz */
    float InvVoxelSize[3], Translation[3];   /* the float copies NanoVDB's Map keeps (mInvMatF diagonal, mVecF) */
} OrcGrid;

typedef struct {                                                             /* PT/PathTracer.h:271-309 subset */
    float ViewInverse[16];        /* column-major */
    float ProjectionInverse[16];
    uint32_t SampleCount;         /* SamplesPerFrame */
    uint32_t MaxDepth;
    float MaxLuminance, FocusDistance, DepthOfFieldStrength;
    float SkyRotationAzimuth, SkyRotationAltitude, EnvironmentIntensity;
    float EmissiveMeshSamplingPDFBias;
    uint32_t ScreenSplitCount;
    /* shader #defines, PT/PathTracer.cpp:621-654 */
    uint32_t EnableSkyMIS, EnableMeshMIS, ShowEnvMapDirectly, UseOnlyGeometryNormals, UseEnergyCompensation, FurnaceTestMode;
    /* volumes: SH/RayGen.slang:162-380, SH/Volume.slang (homogeneous part); PHASE_FUNCTION_* define, PT/PathTracer.cpp:639-650 */
    uint32_t PhaseFunction;       /* 0 Henyey-Greenstein, 1 Draine, 2 Henyey-Greenstein + Draine (PT/PathTracer.h:76-81) */
    uint32_t VolumesCount;
    const OrcVolume *Volumes;
    /* atmosphere: ENABLE_ATMOSPHERE define (PT/PathTracer.cpp:636-637) + UBO fields SH/Bindings.slang:26-37, defaults PT/PathTracer.h:221-232 */
    uint32_t EnableAtmosphere; uint32_t _padA;
    float PlanetPosition[3], PlanetRadius, AtmosphereHeight;
    float RayleighScatteringCoefficientMultiplier[3], MieScatteringCoefficientMultiplier[3], OzoneAbsorptionCoefficientMultiplier[3];
    float RayleighDensityFalloff, MieDensityFalloff, OzoneDensityFalloff, OzonePeak;
    float SunColor[3];
    uint32_t GridCount;
    const OrcGrid *Grids;         /* heterogeneous density data, indexed by OrcVolume::DensityDataIndex */
} OrcConfig;

typedef struct { uint64_t paths, segments, surface_hits, misses, shadow_rays, medium_events; } OrcCounters;   /* medium_events: scattering events inside a mesh medium or an AABB volume */

typedef struct OrcScene OrcScene;

/* AddDensityDataToVolume after the file read (PT/PathTracer.cpp:1391-1452): MaxDensityInTheGrid, the AABB corners, the 32^3 majorant grid, and the
 * temperature patch (normalised temperature overwrites the density value wherever it is positive -- the shader samples emission from the DENSITY
 * buffer, SH/Volume.slang:235-236).  values: Dim.x*Dim.y*Dim.z floats, patched in place; temperature may be NULL. */
void orc_prepare_density_grid(const int32_t indexMin[3], const uint32_t dim[3], float *values, const float *temperature, float temperatureMin, float temperatureMax,
                              float *maxDensities32, float cornerMin[3], float cornerMax[3], float *maxDensityInTheGrid);
/* ---- KAT helpers ---- */
float orc_grid_transmittance(const OrcConfig *cfg, uint32_t seed, const float o[3], const float d[3], float rayDepth);   /* CalculateVolumesTransmittance, one walk */
void orc_volume_walks(const OrcConfig *cfg, uint32_t n, const float *org, const float *dir, const uint32_t *seeds, float rayDepth,
                      float *T, float *scatter, int32_t *vol, uint32_t *rng2);                                          /* both walks on given rays / seeds */
float orc_grid_sample(const OrcConfig *cfg, uint32_t volume, uint32_t seed, const float x[3]);                           /* SampleNanoVDBBuffer */
void orc_blackbody(float kelvin, float out[3]);
float orc_atm_transmittance(const OrcConfig *cfg, uint32_t seed, const float o[3], const float d[3], int channel);      /* CalculateTransmittanceThroughAtmosphere, one walk */
void orc_atm_samples(const OrcConfig *cfg, uint32_t seed, const float incident[3], float rayleigh_dir[3], float sun_dir[3], float sun_color_pdf[4]);   /* SampleRayleigh, SampleSunDisk */                                                                         /* SH/RTCommon.slang:139-172 */
uint32_t orc_pcg_hash(uint32_t seed);                                  /* SH/Sampler.slang:4-9 */
void     orc_rng_floats(uint32_t seed, uint32_t n, float *out);        /* SH/Sampler.slang:38-43 */
float    orc_dielectric_fresnel(float cosI, float eta);                /* SH/Material.slang:434-449 */
void     orc_aces_fitted(const float in[3], float out[3]);             /* SH/PostProcess/Tonemap.slang:20-55 */

/* one texel of the reference's energy-compensation LUT baker (SH/LookupReflect.slang, SH/LookupRefract.slang) */
float    orc_bake_reflect_texel(uint32_t tx, uint32_t ty, uint32_t tz, uint32_t samples, uint32_t seed);
void orc_draine_cos_theta(float rx, float g, float a, float *cos32, double *cos64);
float orc_bake_reflect_params(float viewCosine, float roughness, float anisotropy, float lz_min, uint32_t samples, uint32_t seed);
float    orc_bake_refract_texel(uint32_t tx, uint32_t ty, uint32_t tz, int above_surface, uint32_t samples, uint32_t seed);
float    orc_bake_lut_texel(int kind, uint32_t SX, uint32_t SY, uint32_t SZ, uint32_t tx, uint32_t ty, uint32_t tz, uint32_t sample_count, uint32_t seed);

/* ---- host-side one-offs ---- */
/* PT/PathTracer.cpp:1137-1332. rgba is modified in place (alpha <- pdf). Returns importance sum. */
float orc_build_env_alias(float *rgba, uint32_t w, uint32_t h, OrcAliasEntry *alias_out);
/* PT/Editor.cpp:45-48,1042-1051 + PT/FlyCamera.cpp:84-140: the matrices the shader really receives. */
void  orc_camera_from_view(const float view[16], float aspect, float viewInv_out[16], float projInv_out[16]);
void  orc_default_config(OrcConfig *cfg);
/* Radiance .hdr -> float RGBA (alpha 1), stbi_loadf semantics; free with orc_free. NULL on error. */
float *orc_load_hdr(const char *path, uint32_t *w_out, uint32_t *h_out);
void   orc_free(void *p);

/* ---- scene ---- */
OrcScene *orc_scene_create(const OrcSceneDesc *desc);   /* copies nothing: desc arrays must outlive the scene */
void      orc_scene_destroy(OrcScene *s);
uint32_t  orc_scene_triangle_count(const OrcScene *s);
uint32_t  orc_scene_emissive_count(const OrcScene *s);
/* world-space triangles in (instance, primitive) order: 9 floats each */
void      orc_scene_world_triangles(const OrcScene *s, float *out9, uint32_t *inst_out, uint32_t *prim_out);

/* closest hit, semantics of SH/RTCommon.slang:47-117 / TraceRay (tmin < t < tmax, no culling, ties -> lowest id).
 * use_bvh=0 -> brute force over all triangles. miss: t=-1, prim=inst=0xFFFFFFFF. */
void orc_trace_closest(const OrcScene *s, uint32_t n, const float *org3, const float *dir3, float tmin, float tmax,
                       int use_bvh, float *t_out, uint32_t *prim_out, uint32_t *inst_out, float *uv_out2);

/* One hit's shading step, as closest_hit runs it (SH/ClosestHit.slang:40-238) but without the shadow rays: record i is the hit of
 * instance inst[i], primitive prim[i] at barycentrics uv2[2i..], reached along dir3 from org3 with BSDF pdf pay_pdf[i] at Depth 1, outside
 * any medium, drawing from rng[i].  The sky draw, the light draw and the BSDF draw are made in that order; each drawn direction is
 * evaluated with EvaluateBSDF, and the NEE term c is the one the shader adds when the shadow ray is unoccluded.  L3 (optional): one more
 * world-space direction per record to evaluate.  out: n records of ORC_SQ_STRIDE floats, laid out like B200PT_SQ_* of include/b200pt.h
 * (vectors in tangent space unless named otherwise; LIGHT_GID and RNG hold u32 bits). */
#define ORC_SQ_N          0    /* shading normal, world */
#define ORC_SQ_T          3
#define ORC_SQ_B          6
#define ORC_SQ_NG         9    /* geometry normal, world */
#define ORC_SQ_INSIDE     12
#define ORC_SQ_AX         13
#define ORC_SQ_AY         14
#define ORC_SQ_ETA        15
#define ORC_SQ_PM         16
#define ORC_SQ_PD         17
#define ORC_SQ_PG         18
#define ORC_SQ_BASECOLOR  19
#define ORC_SQ_ROUGHNESS  22
#define ORC_SQ_V          23
#define ORC_SQ_H          26
#define ORC_SQ_EMITTED    29   /* emission term */
#define ORC_SQ_SKY_L      32
#define ORC_SQ_SKY_LV     35   /* radiance, pdf */
#define ORC_SQ_SKY_EVAL   39   /* BxDF, PDF */
#define ORC_SQ_SKY_C      43
#define ORC_SQ_LIGHT_L    46
#define ORC_SQ_LIGHT_LV   49
#define ORC_SQ_LIGHT_EVAL 53
#define ORC_SQ_LIGHT_C    57
#define ORC_SQ_LIGHT_GID  60
#define ORC_SQ_BSDF_L     61   /* 0 when the direction is invalid */
#define ORC_SQ_BSDF_EVAL  64
#define ORC_SQ_VALID      68
#define ORC_SQ_SCATTER    69   /* world */
#define ORC_SQ_SAMPLE     72   /* BxDF, PDF after the geometry-normal rejection */
#define ORC_SQ_REFRACTED  76
#define ORC_SQ_ENTERED    77
#define ORC_SQ_REJECTED   78
#define ORC_SQ_USER_L     79
#define ORC_SQ_USER_EVAL  82
#define ORC_SQ_RNG        86
#define ORC_SQ_CLASS      87   /* GPU only: the material class whose kernel ran */
#define ORC_SQ_POS        88   /* shading position, world */
#define ORC_SQ_SKY_W      91   /* sky draw direction, world */
#define ORC_SQ_LIGHT_W    94   /* light draw direction, world */
#define ORC_SQ_STRIDE     97
void orc_shade_query(const OrcScene *s, const OrcConfig *cfg, uint32_t n, const uint32_t *inst, const uint32_t *prim, const float *uv2, const float *dir3,
                     const float *org3, const float *pay_pdf, const uint32_t *rng, const float *L3, float *out);
/* Miss shading (miss_shader, SH/Miss.slang:8-76) for n world directions dir3 at path depth depth[i] with BSDF pdf pay_pdf[i]: out holds n records
 * of ORC_MQ_STRIDE floats laid out like B200PT_MQ_* of include/b200pt.h (emitted RGB, sky sampler pdf of the lookup). */
#define ORC_MQ_RGB        0
#define ORC_MQ_PDF        3
#define ORC_MQ_STRIDE     4
void orc_miss_query(const OrcScene *s, const OrcConfig *cfg, uint32_t n, const float *dir3, const uint32_t *depth, const float *pay_pdf, float *out);
/* One segment of the path loop (path_segment, SH/RayGen.slang:66-113) and the fold of a finished path into its sample slot (fold_sample,
 * :116-128) for n caller-given paths, laid out like B200PT_BQ_* of include/b200pt.h: the sample slot of record i is i, flags ORC_BQ_STORE /
 * ORC_BQ_CARRY as B200PT_BQ_STORE / CARRY.  Throughput and pathLight travel in the record.  *survivors: the number alive.  Scenes without
 * volumes or the atmosphere. */
#define ORC_BQ_STORE       2
#define ORC_BQ_CARRY       4
#define ORC_BQ_IN_ORG      0
#define ORC_BQ_IN_PDF      3
#define ORC_BQ_IN_DIR      4
#define ORC_BQ_IN_RNG      7
#define ORC_BQ_IN_THR      8
#define ORC_BQ_IN_DFLAGS   11
#define ORC_BQ_IN_RAD      12
#define ORC_BQ_IN_SLOT     15
#define ORC_BQ_IN_MEDIUM   16
#define ORC_BQ_IN_MEDIUM_G 20
#define ORC_BQ_IN_SAMPLE   21
#define ORC_BQ_IN_STRIDE   25
#define ORC_BQ_OUT_T       0
#define ORC_BQ_OUT_U       1
#define ORC_BQ_OUT_V       2
#define ORC_BQ_OUT_INST    3
#define ORC_BQ_OUT_PRIM    4
#define ORC_BQ_OUT_ALIVE   5
#define ORC_BQ_OUT_NEXT    6
#define ORC_BQ_OUT_SAMPLE  27
#define ORC_BQ_OUT_CARRY   31
#define ORC_BQ_OUT_STRIDE  32
void orc_bounce_query(const OrcScene *s, const OrcConfig *cfg, uint32_t n, const float *in, uint32_t flags, float *out, uint32_t *survivors);

/* One reference dispatch sequence: frames [frame0, frame0+nframes) with Seed_f = PCG_HASH(base_seed + f)
 * (SURVEY 8d; the reference's own seed is wall-clock, PT/PathTracer.cpp:127-140), running-mean accumulate
 * into image (RGBA32F, W*H*4) exactly as SH/RayGen.slang:130-159.  Only rows y with
 * ((y / band_rows) % world) == rank are rendered (image-tile partition, SURVEY 8e); pass world=1 for all.
 * nthreads<=0 -> hardware concurrency. */
void orc_render(const OrcScene *s, const OrcConfig *cfg, uint32_t W, uint32_t H,
                uint32_t frame0, uint32_t nframes, uint32_t base_seed,
                uint32_t rank, uint32_t world, uint32_t band_rows,
                float *image, int nthreads, OrcCounters *counters);

/* Single path sample of pixel (x,y) for frame seed `seed` (push-constant Seed): returns pathLight of the
 * first of SampleCount samples; used by fine-grained parity tests. */
void orc_sample_pixel(const OrcScene *s, const OrcConfig *cfg, uint32_t W, uint32_t H,
                      uint32_t x, uint32_t y, uint32_t seed, float out_rgb[3], uint32_t *segments_out);

/* ---- post chain: PT/PostProcessor.cpp:128-246 + SH/PostProcess/{Bloom,Tonemap}.slang ---- */
typedef struct { float Exposure, Gamma, BloomThreshold, BloomStrength, FalloffRange; uint32_t MipCount; } OrcPostConfig;
void     orc_default_post_config(OrcPostConfig *c);
uint32_t orc_bloom_mip_sizes(uint32_t W, uint32_t H, uint32_t *wh_out20); /* returns level count (<=10) */
/* hdr: W*H*4 float; ldr_out: W*H*4 u8; bloom0_out (optional, W*H*4 float) = mip 0 after the up pass */
void     orc_post_process(const float *hdr, uint32_t W, uint32_t H, const OrcPostConfig *c,
                          uint8_t *ldr_out, float *bloom0_out, int nthreads);

#ifdef __cplusplus
}
#endif
#endif
