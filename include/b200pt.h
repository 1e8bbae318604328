/*
 * b200pt.h -- C-ABI of the H100-native wavefront path tracer (libb200pt.so).
 *
 * Drop-in boundary for ONE hot path of Zydak/Vulkan-Path-Tracer: the Monte-Carlo integrator
 * (ray-gen -> traverse -> closest-hit/miss shading -> accumulate) plus the bloom + tonemap post chain.
 * The reference has no FFI; the seam is the C++ class surface its Editor consumes, so every entry point
 * below names the reference member it replaces (paths relative to the reference repository).
 * INTEGRATION.md shows the adapter a maintainer would put behind PathTracer/PostProcessor.
 *
 * Conventions
 *   - every call returns int32 (VHResult-compatible: 0 = OK, negative = error; VulkanHelper/Include/Core/Error.h:14-72),
 *     never aborts, never throws across the boundary.
 *   - one opaque handle == one GPU == one reference `PathTracer` + `PostProcessor` pair; a handle is not
 *     thread-safe (the reference is single-threaded, PathTracer/Editor.cpp:85-89); distinct handles are independent.
 *   - plain pointers + sizes only; matrices are column-major float[16] (glm); images are row 0 first, tightly packed.
 *   - the library copies everything it needs during the call (as PathTracer::SetScene does, PathTracer.cpp:166-167).
 */
#ifndef B200PT_H
#define B200PT_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- result codes (VHResult-compatible subset) ---- */
#define B200PT_OK                     0
#define B200PT_ERR_UNKNOWN           -1
#define B200PT_ERR_INIT_FAILED       -3      /* VK_ERROR_INITIALIZATION_FAILED: file/scene import failed */
#define B200PT_ERR_OUT_OF_MEMORY     -2
#define B200PT_ERR_WRONG_ARGUMENTS   -15000  /* custom range of Error.h */
#define B200PT_ERR_NOT_IMPLEMENTED   -15001  /* reading .vdb files (needs OpenVDB): b200pt_add_density_data_to_volume */
#define B200PT_ERR_NO_SCENE          -15002
#define B200PT_ERR_CUDA              -15003
#define B200PT_ERR_NO_DEVICE         -15004  /* no CUDA device: the product has no CPU fallback */

typedef struct b200pt_s *b200pt_handle;

/* ---- data layouts (sizes asserted in the implementation) ---- */
typedef struct { float Position[3]; float Normal[3]; float TexCoord[2]; } b200pt_vertex;   /* 32 B: Asset.h:16-21, Bindings.slang:7-12 */

typedef struct {                                                                            /* 112 B: PathTracer.h:12-34 */
    float BaseColor[3], EmissiveColor[3], SpecularColor[3], MediumColor[3], MediumEmissiveColor[3];
    float Metallic, Roughness, IOR, Transmission, Anisotropy, AnisotropyRotation;
    float MediumDensity, MediumAnisotropy;
    uint32_t BaseColorTextureIndex, NormalTextureIndex, RoughnessTextureIndex, MetallicTextureIndex, EmissiveTextureIndex;
} b200pt_material;

typedef struct { const b200pt_vertex *vertices; const uint32_t *indices; uint32_t vertex_count, index_count; } b200pt_mesh; /* Asset.h:23-49 */
typedef struct { float Transform[16]; uint32_t MeshIndex, MaterialIndex; } b200pt_instance;                                /* Asset.h:124-129 */
typedef struct { uint32_t width, height, channels, _pad; const uint8_t *data; } b200pt_texture; /* RGBA8 (4) or R8 (1); PathTracer.cpp:812-869 */

typedef struct {                                   /* what PathTracer::SetScene keeps of a SceneAsset (Asset.h:131-138) */
    const b200pt_mesh *meshes;           uint32_t mesh_count, _p0;
    const b200pt_material *materials;    uint32_t material_count, _p1;
    const b200pt_texture *textures;      uint32_t texture_count, _p2;
    const b200pt_instance *instances;    uint32_t instance_count, _p3;
    float camera_view[16];               /* CameraAsset::ViewMatrix */
    float camera_aspect;                 /* CameraAsset::AspectRatio */
    uint32_t _p4;
} b200pt_scene_desc;

typedef struct {                                   /* PathTracer.h:197-233 members behind the ~45 setters */
    uint32_t SamplesPerFrame;            /* SetSamplesPerFrame   (default 1)   */
    uint32_t MaxDepth;                   /* SetMaxDepth          (200)         */
    float    MaxLuminance;               /* SetMaxLuminance      (500)         */
    float    FocusDistance;              /* SetFocusDistance     (1)           */
    float    DepthOfFieldStrength;       /* SetDepthOfFieldStrength (0)        */
    float    SkyRotationAzimuth;         /* SetSkyAzimuth  (deg, 0)            */
    float    SkyRotationAltitude;        /* SetSkyAltitude (deg, 0)            */
    float    SkyIntensity;               /* SetSkyIntensity      (1)           */
    float    EmissiveMeshSamplingPDFBias;/* SetEmissiveMeshSamplingPDFBias (0) */
    uint32_t ScreenChunkCount;           /* SetSplitScreenCount  (1)           */
    uint32_t EnableSkyMIS;               /* SetSkyMIS            (1)           */
    uint32_t EnableMeshMIS;              /* SetMeshMIS           (1)           */
    uint32_t ShowEnvMapDirectly;         /* SetEnvMapShownDirectly (1)         */
    uint32_t UseOnlyGeometryNormals;     /* SetUseOnlyGeometryNormals (0)      */
    uint32_t UseEnergyCompensation;      /* SetUseEnergyCompensation (1)       */
    uint32_t FurnaceTestMode;            /* SetFurnaceTestMode   (0)           */
    uint32_t MaxSamplesAccumulated;      /* SetMaxSamplesAccumulated (5000)    */
    /* engine knobs (no reference equivalent) */
    uint32_t FramesInFlight;             /* frames batched into one wavefront (0 = auto) */
} b200pt_config;

typedef struct { float Exposure, Gamma; } b200pt_tonemap;                               /* PostProcessor.h:8-12  */
typedef struct { float BloomThreshold, BloomStrength; uint32_t MipCount; float FalloffRange; } b200pt_bloom; /* PostProcessor.h:14-21 */

typedef struct {                                   /* device counters + event timings of the last path_trace call */
    uint64_t paths, extend_rays, shade_invocations, surface_hits, misses, shadow_rays, medium_events;
    uint64_t kernel_launches;
    float ms_total, ms_raygen, ms_extend, ms_shade, ms_connect, ms_resolve;
    uint32_t waves, bounces;
} b200pt_counters;

/* ---- lifetime: PathTracer::New / PostProcessor::New (PathTracer.h:83, PostProcessor.h:25) ---- */
int32_t b200pt_create(int32_t device_ordinal, b200pt_handle *out);
int32_t b200pt_destroy(b200pt_handle h);
const char *b200pt_last_error(b200pt_handle h);         /* human-readable detail of the last failure (VH_LOG_ERROR analogue) */
const char *b200pt_version(void);

/* ---- scene: PathTracer::SetScene(const std::string&) (PathTracer.cpp:158-676) ---- */
int32_t b200pt_set_scene_file(b200pt_handle h, const char *gltf_path);      /* glTF 2.0 (.gltf + .bin + PNG/JPEG textures) */
int32_t b200pt_set_scene_arrays(b200pt_handle h, const b200pt_scene_desc *desc);
/* PathTracer::SetEnvMapFilepath / LoadEnvironmentMap (PathTracer.cpp:1048-1056,1137-1332): builds the alias table */
int32_t b200pt_set_env_map_file(b200pt_handle h, const char *hdr_path);
int32_t b200pt_set_env_map(b200pt_handle h, uint32_t width, uint32_t height, const float *rgba);
/* PathTracer::LoadLookupTable x3 (PathTracer.cpp:199-201,871-937): fp32 [32][64][64], [32][128][128] x2 */
int32_t b200pt_set_luts(b200pt_handle h, const float *reflection, const float *refraction_from_outside, const float *refraction_from_inside);
int32_t b200pt_set_luts_dir(b200pt_handle h, const char *dir);              /* dir holding the three shipped .bin files */

/* ---- parameters: the setter/getter block of PathTracer.h:97-181 ---- */
int32_t b200pt_default_config(b200pt_config *out);
int32_t b200pt_set_config(b200pt_handle h, const b200pt_config *cfg);       /* any change -> ResetPathTracing() */
int32_t b200pt_get_config(b200pt_handle h, b200pt_config *out);
int32_t b200pt_material_count(b200pt_handle h, uint32_t *out);
int32_t b200pt_get_material(b200pt_handle h, uint32_t index, b200pt_material *out);   /* GetMaterial */
int32_t b200pt_set_material(b200pt_handle h, uint32_t index, const b200pt_material *m); /* SetMaterial (PathTracer.cpp:712-810) */
int32_t b200pt_get_material_name(b200pt_handle h, uint32_t index, char *buf, uint32_t buf_size); /* GetMaterialName */
/* ---- instance transforms: TLAS::Update (VulkanHelper/Include/Vulkan/TLAS.h:78-85, Source/Vulkan/TLASImpl.cpp:192-293) ----
 * transforms: count x 16 floats, column-major, the layout of b200pt_instance.Transform, in InstanceIndex order; only rows 0-2 are used.
 * The update replaces every instance transform -> ResetPathTracing(); camera, config, image size, partition, materials, volumes and the
 * environment stay.  rebuild == 0 refits the tree in place (same topology, boxes recomputed on the GPU); rebuild == B200PT_REBUILD_GPU builds
 * a new tree on the GPU (PLOC clustering over the LBVH's references, milliseconds, close to the SAH tree's quality; B200PT_BVH_SAH not read);
 * any other nonzero value builds the tree b200pt_set_scene_arrays would build for these transforms (B200PT_BVH_SAH honoured, host passes).
 * Both rebuilds re-choose the traversal shape and launch configuration.
 * WRONG_ARGUMENTS: count != instance count, a null pointer or a non-finite entry; NO_SCENE without a scene.  A rejected call changes
 * nothing.  A failed update restores the previous transforms: a failed rebuild keeps the previous tree, a failed refit refits the tree back
 * to them (if that fails too, the handle reports NO_SCENE until the next set_scene).  The image equals that of a handle loaded with the
 * moved scene. */
int32_t b200pt_instance_count(b200pt_handle h, uint32_t *out);
int32_t b200pt_get_instance_transforms(b200pt_handle h, float *transforms, uint32_t count);
#define B200PT_REBUILD_GPU 2
int32_t b200pt_update_instance_transforms(b200pt_handle h, const float *transforms, uint32_t count, int32_t rebuild);
/* ---- mesh vertices (no reference equivalent: its BLAS are built once in SetScene) ----
 * One call replaces the whole vertex array (position, normal, UV) of each listed mesh; every instance of an updated mesh changes.  Indices and
 * vertex counts stay: vertex_count must equal the mesh's count.  The batch gets one tree update: rebuild has the meaning it has in
 * b200pt_update_instance_transforms (0 refits, B200PT_REBUILD_GPU builds on the GPU, any other value builds what set_scene builds).  The
 * update waits for the waves in flight and resets the accumulation (ResetPathTracing); camera, config, image size, partition, materials,
 * volumes, environment and instance transforms stay.
 * vertices_are_device != 0: every update's vertices pointer is device memory of the handle's GPU, read on the handle's stream.  The caller
 * orders its own writes of those buffers before the call: by synchronising the stream that wrote them, or by writing them on the stream given
 * to b200pt_set_stream.  The buffers are staged and checked on the device; nothing is committed before the check passes.
 * WRONG_ARGUMENTS: a null pointer, n_updates == 0, a mesh index out of range or repeated, a count mismatch or a non-finite component;
 * NO_SCENE without a scene.  A rejected call changes nothing.  A failed update restores the previous vertices: a failed rebuild keeps the
 * previous tree, a failed refit refits the tree back (if that fails too, the handle reports NO_SCENE until the next set_scene).  The image
 * equals that of a handle loaded with the deformed scene. */
typedef struct { uint32_t mesh; uint32_t vertex_count; const b200pt_vertex *vertices; } b200pt_mesh_update;
int32_t b200pt_mesh_count(b200pt_handle h, uint32_t *out);
int32_t b200pt_mesh_vertex_count(b200pt_handle h, uint32_t mesh, uint32_t *out);
int32_t b200pt_get_mesh_vertices(b200pt_handle h, uint32_t mesh, b200pt_vertex *out, uint32_t count);   /* count must equal the mesh's */
int32_t b200pt_update_mesh_vertices(b200pt_handle h, const b200pt_mesh_update *updates, uint32_t n_updates,
                                    int32_t vertices_are_device, int32_t rebuild);
/* ---- glTF animation: node animations, skins and morph targets posed on the GPU (no reference equivalent) ----
 * A scene loaded from a glTF file keeps its node graph, skins (joints, inverseBindMatrices), the JOINTS_n / WEIGHTS_n sets and the morph
 * targets (POSITION / NORMAL / TEXCOORD_0 deltas; TANGENT and COLOR_n are ignored) of its primitives, and its animations.  None of it changes
 * what the load returns; malformed animation data never fails the load and is reported by the pose that needs it.
 * b200pt_pose samples every channel of animation `animation` at `time` as glTF 2.0 Appendix C defines it (time clamped to each sampler's
 * keys; STEP, LINEAR with slerp for rotations, CUBICSPLINE), in double rounded to float; animation == -1 is the rest pose (the nodes' own
 * TRS, default morph weights: node.weights, else mesh.weights, else 0; skins applied).  Node world matrices use the loader's arithmetic, so a
 * node no channel touches keeps its load-time instance transform bit for bit.  Skinned meshes follow the spec: the skinned node's transform
 * is ignored, the vertices are posed in glTF world space (joint matrix = world(joint) x inverseBind) and their instances get the
 * y flip diag(1, -1, 1, 1) as transform.  Vertices are computed from the rest data on the GPU, never from the previous pose, so a pose
 * depends only on (file, animation, time).  Every instance transform and the vertices of every mesh some skin or morph target touches are
 * replaced, whatever b200pt_update_instance_transforms / b200pt_update_mesh_vertices set before; other meshes keep theirs.  One tree update
 * per pose, rebuild as in b200pt_update_instance_transforms; the pose waits for the waves in flight and resets the accumulation.
 * WRONG_ARGUMENTS: an animation index out of range, a non-finite time, malformed animation data the pose needs (indices out of range, count
 * mismatches, keys that do not increase, non-finite values, a non-finite posed vertex), or a mesh its instances would deform two ways
 * (different skins or weights, or skinned and not); b200pt_last_error names the problem.  NO_SCENE without a scene, or for a scene without
 * glTF node data (OBJ, b200pt_set_scene_arrays).  A rejected pose changes nothing; a failed update restores the previous state as
 * b200pt_update_mesh_vertices does.  The image equals that of a handle loaded with the posed vertices and transforms. */
int32_t b200pt_animation_count(b200pt_handle h, uint32_t *out);
int32_t b200pt_get_animation(b200pt_handle h, uint32_t index, char *name, uint32_t name_len, float *t0, float *t1);   /* t0 / t1: first and last key time */
int32_t b200pt_pose(b200pt_handle h, int32_t animation, float time, int32_t rebuild);
/* host halves (test hooks, no GPU needed), on a glTF file: the animation count and, for index < count, its name and key range; and the
 * pose's node world matrices (glTF world space, column-major, 16 floats per node) and per-node morph weights (weight_counts[node] floats each,
 * concatenated in node order).  With world == NULL only node_count and weights_total are written. */
int32_t b200pt_gltf_animation_info(const char *path, int32_t index, uint32_t *count, char *name, uint32_t name_len, float *t0, float *t1);
int32_t b200pt_gltf_pose_nodes(const char *path, int32_t animation, float time, uint32_t *node_count, float *world, uint32_t *weight_counts,
                               float *weights, uint32_t *weights_total);
int32_t b200pt_set_camera(b200pt_handle h, const float view_inverse[16], const float projection_inverse[16]); /* SetCameraViewInverse/ProjectionInverse */
int32_t b200pt_get_camera(b200pt_handle h, float view_inverse[16], float projection_inverse[16]);
/* the Editor/FlyCamera round trip that produces the matrices the shader really sees (Editor.cpp:45-48,1042-1051; FlyCamera.cpp:84-140) */
int32_t b200pt_camera_from_view(const float view[16], float aspect, float view_inverse_out[16], float projection_inverse_out[16]);
int32_t b200pt_resize(b200pt_handle h, uint32_t width, uint32_t height);   /* ResizeImage */
int32_t b200pt_get_size(b200pt_handle h, uint32_t *width, uint32_t *height);
int32_t b200pt_reset(b200pt_handle h);                                      /* ResetPathTracing */
/* ---- volumes: PathTracer::AddVolume / RemoveVolume / SetVolume / GetVolumes / SetPhaseFunction / AddDensityDataToVolume /
 * RemoveDensityDataFromVolume (PathTracer.h:36-81,157-166, PathTracer.cpp:1334-1555).  Homogeneous AABB volumes (SH/Volume.slang with
 * m_DensityDataIndex == -1, SH/RayGen.slang:162-380): free-flight sampling against the geometry distance, phase-function scattering with sky /
 * light NEE, analytic transmittance on the NEE terms.  Heterogeneous volumes (SH/Volume.slang:54-166,230-252,291-352,448-517): delta tracking
 * against the 32^3 grid of majorants, ratio-tracked NEE transmittance on the path's own random stream, blackbody / coloured emission from the
 * temperature data -- over a DENSE copy of the values the reference keeps in a NanoVDB buffer (b200pt_add_density_grid_to_volume).  Reading
 * .vdb files needs OpenVDB (a vcpkg dependency of the reference, absent here): b200pt_add_density_data_to_volume returns NOT_IMPLEMENTED, the
 * adapter reads the file with the reference's own OpenVDB and hands the values over (INTEGRATION.md).  At most B200PT_MAX_VOLUMES. */
#define B200PT_MAX_VOLUMES 100   /* the reference sorts into float distances[100] (RayGen.slang:165); also MAX_HETEROGENEOUS_VOLUMES (PathTracer.h:195) */
typedef struct {                         /* PathTracer::Volume, PT/PathTracer.h:36-70 (defaults in comments) */
    float CornerMin[3], CornerMax[3];    /* local AABB (-1 / +1); overwritten by b200pt_add_density_grid_to_volume (PathTracer.cpp:1408-1420) */
    float Position[3], Scale[3];         /* (0 / 1): world AABB = Position + Corner * Scale (VolumeGPU's constructor, PathTracer.h:396-397) */
    float Color[3];                      /* scattering albedo (0.8)            */
    float EmissiveColor[3];              /* (0)                                */
    float TemperatureColor[3];           /* emission colour when UseBlackbody == 0 (1, 0.5, 0) */
    float Density;                       /* extinction coefficient (1); scales the grid values of a heterogeneous volume */
    float Anisotropy;                    /* g of Henyey-Greenstein / Draine (0)*/
    float Alpha;                         /* Draine alpha (1)                   */
    float DropletSize;                   /* HG + Draine fit, micrometres (20)  */
    int32_t DensityDataIndex;            /* READ-ONLY: -1 = homogeneous, else the slot b200pt_add_density_grid_to_volume assigned (PathTracer.cpp:1512-1513); add / set ignore it */
    float MaxDensityInTheGrid;           /* READ-ONLY (PathTracer.cpp:1393-1394) */
    int32_t UseBlackbody;                /* (1) blackbody colour from the Kelvin range, else TemperatureColor */
    int32_t HasTemperatureData;          /* READ-ONLY: the density data came with a temperature grid (PathTracer.h:398) */
    float TemperatureGamma, TemperatureScale, EmissiveColorGamma;   /* (1, 1, 1) */
    int32_t KelvinMin, KelvinMax;        /* (500, 8000) */
    uint32_t ApproximatedScatteringForClouds; /* anisotropy / density decay with the depth (0) */
    float ApproximatedScatteringFalloff; /* (0.8) */
    float GridSharpness;                 /* (1) multiplies the normalised grid value before the clamp to [0, 1] */
} b200pt_volume;
int32_t b200pt_default_volume(b200pt_volume *out);
int32_t b200pt_add_volume(b200pt_handle h, const b200pt_volume *volume);                 /* AddVolume  -> ResetPathTracing() */
int32_t b200pt_set_volume(b200pt_handle h, uint32_t index, const b200pt_volume *volume); /* SetVolume  -> ResetPathTracing(); density data stays attached to the index */
int32_t b200pt_remove_volume(b200pt_handle h, uint32_t index);                           /* RemoveVolume (later volumes move down one index) */
int32_t b200pt_volume_count(b200pt_handle h, uint32_t *out);
int32_t b200pt_get_volume(b200pt_handle h, uint32_t index, b200pt_volume *out);          /* GetVolumes()[index] */
/* Density data of a heterogeneous volume: what AddDensityDataToVolume holds after openvdb::io::File::readGrid (PathTracer.cpp:1361-1406) --
 * the "density" FloatGrid (and "temperature" / "flames") over the density grid's active-voxel bounding box. */
typedef struct {
    int32_t IndexMin[3];                 /* evalActiveVoxelBoundingBox().min() */
    uint32_t Dim[3];                     /* evalActiveVoxelDim() */
    const float *Density;                /* Dim[0]*Dim[1]*Dim[2] floats, x fastest: tree().getValue(IndexMin + (x, y, z)) */
    const float *Temperature;            /* NULL, or the temperature grid's values at the same coordinates */
    float TemperatureMin, TemperatureMax;/* tools::minMax of the temperature grid's active values (PathTracer.cpp:1403-1404); Min >= Max: taken from the array */
    double VoxelSize;                    /* the density grid's index-to-world map: uniform scale ... */
    double Translation[3];               /* ... and translation (identity: 1, {0, 0, 0}) */
} b200pt_density_grid;
int32_t b200pt_add_density_grid_to_volume(b200pt_handle h, uint32_t index, const b200pt_density_grid *grid);   /* AddDensityDataToVolume after the file read (PathTracer.cpp:1391-1515) -> ResetPathTracing() */
int32_t b200pt_add_density_data_to_volume(b200pt_handle h, uint32_t index, const char *vdb_path);   /* AddDensityDataToVolume(filepath): NOT_IMPLEMENTED (needs OpenVDB) */
int32_t b200pt_remove_density_data_from_volume(b200pt_handle h, uint32_t index);                    /* RemoveDensityDataFromVolume (PathTracer.cpp:1518-1528): homogeneous again, corners back to -1 / +1 */
/* host half of b200pt_add_density_grid_to_volume (test hook, no GPU needed): the temperature-patched values, the 32^3 majorants, the AABB corners, MaxDensityInTheGrid */
int32_t b200pt_prepare_density_grid(const b200pt_density_grid *grid, float *values_out, float *max_densities_out, float corner_min[3], float corner_max[3], float *max_density_in_the_grid);
/* ---- atmosphere: the twelve setters / getters of PathTracer.h:129-144,170-181 (members :221-232) as one parameter block; any set ->
 * ResetPathTracing().  Enable != 0 renders with the reference's atmosphere (SH/Atmosphere.slang, SH/RayGen.slang:76-84,212-255,382-471): a miss
 * emits nothing, the sky NEE samples the sun disk (direction from SkyRotationAzimuth / Altitude), Rayleigh / Mie / ozone events are found by delta
 * tracking on one colour channel (the path is split at its first atmosphere event), and sky NEE terms are attenuated by a ratio-tracked
 * transmittance.  Parity-tested against the CPU oracle (tests/test_gpu_parity.py::test_atmosphere_matches_oracle). */
typedef struct {
    uint32_t Enable;                                    /* SetEnableAtmosphere (false)                         */
    float    PlanetPosition[3];                         /* SetPlanetPosition   (0, 6360e3 + 1000, 0) metres    */
    float    PlanetRadius;                              /* SetPlanetRadius     (6360e3)                        */
    float    AtmosphereHeight;                          /* SetAtmosphereHeight (100e3)                         */
    float    RayleighScatteringCoefficientMultiplier[3];/* (1, 1, 1)                                           */
    float    MieScatteringCoefficientMultiplier[3];     /* (1, 1, 1)                                           */
    float    OzoneAbsorptionCoefficientMultiplier[3];   /* (1, 1, 1)                                           */
    float    RayleighDensityFalloff;                    /* (8000)                                              */
    float    MieDensityFalloff;                         /* (1200)                                              */
    float    OzoneDensityFalloff;                       /* (5000)                                              */
    float    OzonePeak;                                 /* (22000)                                             */
    float    SunColor[3];                               /* SetSunColor (1, 0.956, 0.88)                        */
} b200pt_atmosphere;
int32_t b200pt_default_atmosphere(b200pt_atmosphere *out);
int32_t b200pt_set_atmosphere(b200pt_handle h, const b200pt_atmosphere *a);
int32_t b200pt_get_atmosphere(b200pt_handle h, b200pt_atmosphere *out);
/* PathTracer::GetTotalVertexCount / GetTotalIndexCount (PathTracer.h:122-123): summed over the loaded meshes */
int32_t b200pt_get_total_counts(b200pt_handle h, uint64_t *vertex_count_out, uint64_t *index_count_out);
/* PathTracer::SetPhaseFunction (PathTracer.h:76-81,168-169): 0 Henyey-Greenstein, 1 Draine, 2 Henyey-Greenstein + Draine */
int32_t b200pt_set_phase_function(b200pt_handle h, uint32_t phase_function);
int32_t b200pt_get_phase_function(b200pt_handle h, uint32_t *out);

/* ---- image-tile partition across GPUs (no reference equivalent; SURVEY 8e) ----
 * rank r of `world` owns rows y with ((y / band_rows) % world) == r.  RNG streams are keyed on global pixel
 * coordinates, so the union of all ranks' rows is bit-identical to the world==1 image. */
int32_t b200pt_set_partition(b200pt_handle h, uint32_t rank, uint32_t world, uint32_t band_rows);
int32_t b200pt_local_rows(b200pt_handle h, uint32_t *rows_out);
/* pure host helper: global row of local row `r` (also used by the gather step) */
uint32_t b200pt_partition_global_row(uint32_t local_row, uint32_t rank, uint32_t world, uint32_t band_rows);
uint32_t b200pt_partition_local_row_count(uint32_t height, uint32_t rank, uint32_t world, uint32_t band_rows);

/* ---- the hot path: PathTracer::PathTrace(cmd) x `dispatches` (PathTracer.cpp:122-156) ----
 * dispatch d uses push constants {FrameCount = floor(d/S^2), Seed = PCG_HASH(base_seed + d), ChunkIndex = d % S^2}
 * (the reference's wall-clock seed is replaced by a caller-supplied one).  Stops early at MaxSamplesAccumulated;
 * *done_out (optional) = 1 when all samples are accumulated (PathTrace's return value). */
int32_t b200pt_path_trace(b200pt_handle h, uint32_t dispatches, uint32_t base_seed, int32_t *done_out);
int32_t b200pt_samples_accumulated(b200pt_handle h, uint32_t *out);         /* GetSamplesAccumulated */

/* ---- adaptive sampling (no reference equivalent) ----
 * With Enable != 0 every local pixel keeps its frame count n_p and a Welford running mean / second moment of its per-frame luminance
 * (acc / SamplesPerFrame, weights 0.212671 0.715160 0.072169).  Whenever the frame counter reaches a multiple of Interval, a pixel with
 * n_p >= MinSamples stops for good once sqrt(M2 / (n_p - 1) / n_p) <= Threshold * max(mean, 1e-3) (Threshold 0 stops nothing).  Pixels
 * are traced from frame 0 until they stop, so a stopped pixel holds bit for bit what the plain renderer holds after n_p frames.
 * path_trace then also returns done once no local pixel is active, and launches nothing.  MaxSamplesAccumulated stays the cap.
 * Not combinable with ScreenChunkCount > 1.  Any set resets the accumulation; so do reset / set_config / resize / set_partition. */
typedef struct { uint32_t Enable; float Threshold; uint32_t MinSamples; uint32_t Interval; } b200pt_adaptive;   /* defaults {0, 0.01, 64, 32} */
int32_t b200pt_default_adaptive(b200pt_adaptive *out);
int32_t b200pt_set_adaptive(b200pt_handle h, const b200pt_adaptive *a);   /* WRONG_ARGUMENTS: Threshold < 0 or not finite, MinSamples < 2, Interval 0, chunks > 1 */
int32_t b200pt_get_adaptive(b200pt_handle h, b200pt_adaptive *out);
/* local rows: counts[i] = frames accumulated into pixel i (the frame count everywhere without adaptive sampling), rel_error[i] = its
 * sqrt(M2 / (n_p - 1) / n_p) / max(mean, 1e-3) (NaN without adaptive sampling or with n_p < 2).  Either pointer may be NULL. */
int32_t b200pt_get_pixel_stats(b200pt_handle h, uint32_t *counts, float *rel_error);
int32_t b200pt_active_pixels(b200pt_handle h, uint32_t *out);             /* local pixels still traced (all of them without adaptive sampling) */
/* Per-pixel statistics without adaptive sampling: with enable != 0 the handle keeps the same per-pixel records as adaptive sampling
 * (frame count, Welford mean / M2 of the per-frame luminance) for every local pixel, but takes no decisions: every pixel is traced in every
 * frame, and the image and the work counters are bit-identical to a run without statistics.  b200pt_get_pixel_stats then reports rel_error,
 * and checkpoints use version 2 (the adaptive block as set, then the records).  With adaptive sampling on, its records are the statistics.
 * Not combinable with ScreenChunkCount > 1.  Any set resets the accumulation, as b200pt_set_adaptive does. */
int32_t b200pt_set_track_variance(b200pt_handle h, int32_t enable);
int32_t b200pt_get_track_variance(b200pt_handle h, int32_t *out);

/* ---- denoiser (no reference equivalent; DESIGN.md section 12) ----
 * An a-trous wavelet filter (Dammertz et al. 2010) with the edge-stopping weights of SVGF (Schied et al. 2017) on the albedo-demodulated
 * accumulation, guided by per-pixel features of the first surface seen through the pixel and by the variance of the pixel's mean luminance.
 * Features: FeatureSamples camera rays per pixel (jitter and depth of field as the render), closest hit only (volumes and the atmosphere are
 * not seen).  albedo_cov = (mean albedo (pd + pm) * BaseColor + pg, a miss counting 1; coverage = fraction of rays that hit),
 * normal_depth = (mean world-space shading normal, misses counting 0, not renormalised; mean view depth of the hits, 0 without hits).
 * variance = M2 / (n - 1) / n of the records, 1e30 below two frames.  The denoised image is biased by design; the accumulation stays the
 * reference-matching output.  WRONG_ARGUMENTS: Iterations > 10, FeatureSamples 0 or > 256, a sigma negative or not finite, null pointers. */
typedef struct { uint32_t Iterations; uint32_t FeatureSamples; float SigmaLuminance; float SigmaNormal; float SigmaDepth; } b200pt_denoise_params;   /* defaults {5, 8, 4, 128, 1} */
int32_t b200pt_default_denoise(b200pt_denoise_params *out);
/* feature pass + filter into a denoised RGBA32F W*H image owned by the handle; the accumulation image is not touched.  Needs statistics or
 * adaptive sampling on and world == 1 (WRONG_ARGUMENTS otherwise).  elapsed_ms (optional): device time of the feature pass and the filter. */
int32_t b200pt_denoise(b200pt_handle h, const b200pt_denoise_params *p, float *elapsed_ms);
int32_t b200pt_get_denoised(b200pt_handle h, float *dst_rgba32f, int32_t dst_is_device);   /* W*H*4 floats of the last b200pt_denoise */
/* the filter's inputs for this handle's local rows (any partition; host memory; each pointer may be NULL): albedo_cov and normal_depth
 * local_rows*W*4 floats, variance local_rows*W floats.  Needs statistics or adaptive sampling on.  What an external denoiser is fed, and
 * what a multi-GPU caller gathers to rank 0 for b200pt_denoise_image. */
int32_t b200pt_get_denoise_inputs(b200pt_handle h, const b200pt_denoise_params *p, float *albedo_cov, float *normal_depth, float *variance);
/* the filter alone on caller buffers of a width x height image (all host or all device memory): color / albedo_cov / normal_depth / out
 * RGBA32F, variance one float per pixel.  Iterations == 0 copies color to out bit for bit. */
int32_t b200pt_denoise_image(b200pt_handle h, uint32_t width, uint32_t height, const float *color, const float *albedo_cov, const float *normal_depth,
                             const float *variance, const b200pt_denoise_params *p, float *out, int32_t is_device);
int32_t b200pt_synchronize(b200pt_handle h);
/* b200pt_path_trace is ASYNCHRONOUS: it returns once the waves are enqueued (two waves are in flight on the handle's internal streams so that the
 * latency-bound tail of one overlaps the head of the next, also across calls).  Every later call on the handle that touches the image (get_hdr,
 * post_process, set_hdr, checkpoints, ...) is ordered behind them automatically.  Work the CALLER enqueues on the handle's stream -- its own kernels
 * on b200pt_hdr_device_ptr, a timing event -- needs b200pt_flush first: it makes the stream wait (on the device, no host synchronisation) for
 * everything launched so far.  b200pt_synchronize additionally blocks the host. */
int32_t b200pt_flush(b200pt_handle h);
/* Run all work of this handle on a caller-owned CUDA stream (cudaStream_t passed as void*; NULL = the handle's own
 * stream).  Lets a host framework order its collectives / events against the render without extra synchronisation. */
int32_t b200pt_set_stream(b200pt_handle h, void *cuda_stream);
/* 1 = record CUDA events around every kernel class and report ms_raygen/extend/shade/connect/resolve in the counters
 * (adds a few microseconds per launch; leave 0 for throughput runs). */
int32_t b200pt_set_profiling(b200pt_handle h, int32_t enabled);
/* GetOutputImage(): RGBA32F running mean, alpha 1.  world==1: full W*H*4 floats.  world>1: local rows only
 * (local_rows*W*4 floats, in local-row order).  dst may be host or device memory (dst_is_device). */
int32_t b200pt_get_hdr(b200pt_handle h, float *dst, int32_t dst_is_device);
int32_t b200pt_hdr_device_ptr(b200pt_handle h, void **ptr_out);            /* zero-copy view for the NCCL gather */
/* replace the accumulation image (post-only runs / checkpoint restore): full W*H*4 floats from host or device */
int32_t b200pt_set_hdr(b200pt_handle h, const float *src, int32_t src_is_device);
/* Checkpoint / resume of the progressive accumulation (the reference keeps it only in the GPU image and loses it on exit, PathTracer.h:183,
 * 199-201; SURVEY 5 / 8f row 4).  The file holds the RGBA32F accumulation of THIS handle's rows + the dispatch counters; after
 * b200pt_load_checkpoint into a handle with the same scene / config / size / partition, path_trace(frames, same base_seed) continues the
 * identical sample sequence: the final image equals an uninterrupted run bit for bit.  With adaptive sampling on, the file (version 2) also
 * holds the adaptive block and the per-pixel state; it loads only into a handle with the same adaptive block, and a version-1 file does not. */
int32_t b200pt_save_checkpoint(b200pt_handle h, const char *path);
int32_t b200pt_load_checkpoint(b200pt_handle h, const char *path);
int32_t b200pt_get_counters(b200pt_handle h, b200pt_counters *out);

/* ---- post chain: PostProcessor (PostProcessor.h:25-33, PostProcessor.cpp:128-246) ---- */
int32_t b200pt_post_set_tonemap(b200pt_handle h, const b200pt_tonemap *t);  /* SetTonemappingData */
int32_t b200pt_post_set_bloom(b200pt_handle h, const b200pt_bloom *b);      /* SetBloomData */
int32_t b200pt_post_process(b200pt_handle h);                               /* PostProcess(cmd); input = GetOutputImage() */
int32_t b200pt_post_process_denoised(b200pt_handle h);                      /* the same chain on the image of the last b200pt_denoise */
int32_t b200pt_get_ldr(b200pt_handle h, uint8_t *dst_rgba8, int32_t dst_is_device); /* GetOutputImageView() -> RGBA8 */
/* Multi-GPU post pass (BASELINE config 5; no reference equivalent): PostProcess for output rows [y0, y1) only.  Every rank holds the full HDR input
 * (b200pt_set_hdr) and recomputes the few halo rows of each bloom mip its block depends on, so the rows equal those of b200pt_post_process bit for
 * bit and no exchange is needed before the final gather of the RGBA8 blocks.  b200pt_get_ldr_rows copies rows [y0, y1) (packed, (y1-y0)*W*4 bytes);
 * with a device destination the copy is asynchronous on the handle's stream. */
int32_t b200pt_post_process_rows(b200pt_handle h, uint32_t y0, uint32_t y1);
/* The "HDR accumulate" stage of config 5 as a stand-alone pass (SH/RayGen.slang:130-137; inside b200pt_path_trace the same rule runs in k_resolve):
 * rows [y0, y1) of a full-size RGBA32F frame in DEVICE memory are folded into the accumulation image with lerp(prev, new, 1 / (frame_index + 1)).
 * b200pt_post_input_rows reports which HDR rows b200pt_post_process_rows(y0, y1) reads (block + halo), i.e. the rows a rank has to accumulate. */
int32_t b200pt_accumulate_rows(b200pt_handle h, const float *frame_rgba32f_device, uint32_t frame_index, uint32_t y0, uint32_t y1);
int32_t b200pt_post_input_rows(b200pt_handle h, uint32_t y0, uint32_t y1, uint32_t *in_y0, uint32_t *in_y1);
int32_t b200pt_get_ldr_rows(b200pt_handle h, uint32_t y0, uint32_t y1, uint8_t *dst_rgba8, int32_t dst_is_device);
int32_t b200pt_get_bloom(b200pt_handle h, float *dst_rgba32f);              /* bloom mip 0 after the up pass (test hook) */
int32_t b200pt_bloom_mip_sizes(uint32_t width, uint32_t height, uint32_t *wh_out20, uint32_t *levels_out);
/* Editor::SaveToFile (Editor.cpp:815-843): RGBA8 -> PNG, row stride W*4 */
int32_t b200pt_save_png(b200pt_handle h, const char *path);

/* ---- fine-grained hooks used by the parity tests (closest-hit semantics of RTCommon.slang:47-117) ---- */
/* b200pt_trace_query's closest-hit walk (tmin < t < tmax for every ray, subtract-then-multiply slabs) in the shape the renderer's one-ray-per-thread
 * kernels take for the scene: B200PT_TRAV_FLAT or _SHARED when the BVH is staged in shared memory, _GLOBAL otherwise.  Outputs as there. */
int32_t b200pt_trace_closest(b200pt_handle h, uint32_t n, const float *origins3, const float *directions3,
                             float tmin, float tmax, float *t_out, uint32_t *prim_out, uint32_t *inst_out, float *uv_out2);
/* the volume walks on given rays (parity hook; needs no scene): out_T[i] = Volume::CalculateVolumesTransmittance (SH/Volume.slang:419-446) from seeds[i],
 * out_scatter[i] / out_volume[i] = the free-flight half of ScatteredInVolume (SH/RayGen.slang:164-209: distance or -1, index of the scattering volume
 * or -1) from the same seed, out_rng[2*i] / [2*i+1] = the sampler state after each -- the number of random numbers a walk consumed must match too */
int32_t b200pt_volume_walks(b200pt_handle h, uint32_t n, const float *origins3, const float *directions3, const uint32_t *seeds, float ray_depth,
                            float *out_T, float *out_scatter, int32_t *out_volume, uint32_t *out_rng2);
/* traversal cost of b200pt_trace_closest's walk: nodes_tris_out[2*i] = BVH nodes visited, [2*i+1] = triangles tested (measurement hook) */
int32_t b200pt_trace_stats(b200pt_handle h, uint32_t n, const float *origins3, const float *directions3, float tmin, float tmax, uint32_t *nodes_tris_out);
/* Traversal test hook: ray i (per-ray tmin[i] < t < tmax[i]) through one traversal shape the renderer can launch and one query kind.
 * shape: B200PT_TRAV_SHARED / _GLOBAL: BVH2 stack walk, one ray per thread, BVH staged in shared memory / read from global memory;
 *        _FLAT: the slot-by-slot walk of scenes of at most B200PT_FLAT_MAX triangles; _FIXED_ORIGIN: the same with every ray starting at
 *        origins3[0] (the camera kernel's table; closest-hit only); _DYN2 / _DYN4: the dynamic-fetch kernels over the BVH2 / the BVH4;
 *        _DYN4_SPILL: the BVH4 with a 4-entry shared-memory stack, so the local-memory overflow stack carries the walk.
 * kind:  B200PT_QUERY_CLOSEST: t_out (-1 on a miss), prim_out / inst_out (0xFFFFFFFF on a miss), uv_out2;
 *        B200PT_QUERY_ANY: occluded_out[i] = 1 when some triangle has tmin < t < tmax;
 *        B200PT_QUERY_TARGET: light visibility: a triangle occludes when t < tmax, or when t == tmax and its id (instance-major triangle
 *        index) is below target_gid[i]; tmax_test[i] >= 0 is the acceptance bound of the triangle test (the fused shading kernel passes
 *        nextafter(tmax) for light rays and tmax for sky rays), < 0 takes nextafter(tmax).
 * fma_slabs != 0: the one-FMA slab form of secondary rays instead of subtract-then-multiply.
 * stats3_out (optional): [3*i] nodes visited, [3*i+1] triangles tested, [3*i+2] pushes refused by a full stack.
 * B200PT_ERR_WRONG_ARGUMENTS when the scene has no such shape (no flat walk, no BVH4, BVH too big for shared memory). */
#define B200PT_TRAV_SHARED       0
#define B200PT_TRAV_GLOBAL       1
#define B200PT_TRAV_FLAT         2
#define B200PT_TRAV_FIXED_ORIGIN 3
#define B200PT_TRAV_DYN2         4
#define B200PT_TRAV_DYN4         5
#define B200PT_TRAV_DYN4_SPILL   6
#define B200PT_QUERY_CLOSEST     0
#define B200PT_QUERY_ANY         1
#define B200PT_QUERY_TARGET      2
int32_t b200pt_trace_query(b200pt_handle h, int32_t shape, int32_t kind, int32_t fma_slabs, uint32_t n, const float *origins3, const float *directions3,
                           const float *tmin, const float *tmax, const uint32_t *target_gid, const float *tmax_test,
                           float *t_out, uint32_t *prim_out, uint32_t *inst_out, float *uv_out2, uint32_t *occluded_out, uint32_t *stats3_out);
/* Shading test hook: one shading step of the renderer's hit kernel (k_shade_hit, SH/ClosestHit.slang:40-238) for caller-given hits,
 * through the same device functions and the same class instantiation, without the shadow queries.  Hit i: instance inst[i], primitive
 * prim[i] of that instance's mesh, barycentrics uv2[2i..], world ray direction dir3, ray origin org3 and BSDF pdf pay_pdf[i] of the
 * segment that reached it (the emission MIS term of a hit at Depth > 0), sampler state rng[i].  The sky draw, the light draw and the
 * BSDF draw are made in the renderer's order and each is evaluated; c is the NEE term added when the shadow ray is unoccluded.
 * L3 (optional): one more world direction per hit at which the BSDF is evaluated.  force_general != 0 runs the all-lobes instantiation
 * instead of the triangle's material class.  The current config supplies the rest.  out: n records of B200PT_SQ_STRIDE floats at the
 * offsets below (vectors in tangent space unless marked world; LIGHT_GID and RNG hold u32 bits).  B200PT_ERR_WRONG_ARGUMENTS for an
 * instance or primitive out of range, and for scenes with volumes or the atmosphere on (their paths have walk-level hooks). */
#define B200PT_SQ_N          0    /* shading normal (world) */
#define B200PT_SQ_T          3    /* tangent (world, rotated) */
#define B200PT_SQ_B          6    /* bitangent (world) */
#define B200PT_SQ_NG         9    /* geometry normal (world) */
#define B200PT_SQ_INSIDE     12   /* HitFromInside */
#define B200PT_SQ_AX         13
#define B200PT_SQ_AY         14
#define B200PT_SQ_ETA        15
#define B200PT_SQ_PM         16   /* lobe probabilities */
#define B200PT_SQ_PD         17
#define B200PT_SQ_PG         18
#define B200PT_SQ_BASECOLOR  19
#define B200PT_SQ_ROUGHNESS  22
#define B200PT_SQ_V          23
#define B200PT_SQ_H          26   /* sampled half vector */
#define B200PT_SQ_EMITTED    29   /* emission term */
#define B200PT_SQ_SKY_L      32
#define B200PT_SQ_SKY_LV     35   /* radiance, pdf */
#define B200PT_SQ_SKY_EVAL   39   /* BxDF, PDF */
#define B200PT_SQ_SKY_C      43
#define B200PT_SQ_LIGHT_L    46
#define B200PT_SQ_LIGHT_LV   49
#define B200PT_SQ_LIGHT_EVAL 53
#define B200PT_SQ_LIGHT_C    57
#define B200PT_SQ_LIGHT_GID  60   /* sampled emissive triangle */
#define B200PT_SQ_BSDF_L     61   /* sampled direction, 0 when invalid */
#define B200PT_SQ_BSDF_EVAL  64
#define B200PT_SQ_VALID      68
#define B200PT_SQ_SCATTER    69   /* sampled direction (world) */
#define B200PT_SQ_SAMPLE     72   /* BxDF, PDF after the geometry-normal rejection */
#define B200PT_SQ_REFRACTED  76
#define B200PT_SQ_ENTERED    77   /* refracted into the object: a medium starts */
#define B200PT_SQ_REJECTED   78
#define B200PT_SQ_USER_L     79
#define B200PT_SQ_USER_EVAL  82
#define B200PT_SQ_RNG        86   /* sampler state after the step */
#define B200PT_SQ_CLASS      87   /* material class whose instantiation ran */
#define B200PT_SQ_POS        88   /* shading position (world) */
#define B200PT_SQ_SKY_W      91   /* sky draw direction (world) */
#define B200PT_SQ_LIGHT_W    94   /* light draw direction (world) */
#define B200PT_SQ_STRIDE     97
int32_t b200pt_shade_query(b200pt_handle h, int32_t force_general, uint32_t n, const uint32_t *inst, const uint32_t *prim, const float *uv2,
                           const float *dir3, const float *org3, const float *pay_pdf, const uint32_t *rng, const float *L3, float *out);
/* Miss shading test hook: what the renderer's miss kernel (k_shade_miss, SH/Miss.slang:8-76) gives a path whose segment missed, for n
 * caller-given world directions dir3, path depths depth[i] and BSDF pdfs pay_pdf[i] of the missed segment, under the current config:
 * the environment seen along the direction (inverse sky rotation, lat-long lookup) times the intensity, or the furnace's 1, MIS-weighted
 * at depth > 0 against the sky sampler's pdf.  out: n records of B200PT_MQ_STRIDE floats.  B200PT_ERR_NO_SCENE without a scene or an
 * environment map. */
#define B200PT_MQ_RGB        0    /* emitted radiance */
#define B200PT_MQ_PDF        3    /* sky sampler pdf of the direction (alpha of the lookup; 1 where no lookup is made) */
#define B200PT_MQ_STRIDE     4
int32_t b200pt_miss_query(b200pt_handle h, uint32_t n, const float *dir3, const uint32_t *depth, const float *pay_pdf, float *out);
/* Bounce test hook: one non-primary bounce of the renderer (the extension ray, miss or hit shading, the NEE queries, the path epilogue and the
 * compaction of the survivors) for n caller-given live paths, through the launch sequence and the kernels Engine::path_trace runs for the
 * current scene and config.  in: n records of B200PT_BQ_IN_STRIDE floats; the sample slot of record i is i (IN_SLOT is ignored), IN_SAMPLE is
 * the slot's value before the bounce.  DFLAGS = Depth | (colour channel + 1, 0 = unsplit) << 27 | InMedium << 31.  flags: B200PT_BQ_STORE
 * (a path end stores its radiance instead of adding it to the slot), B200PT_BQ_CARRY (a path end stores its RNG state for a next sub-wave).
 * out: n records of B200PT_BQ_OUT_STRIDE floats, record i for input i: the hit of the extension ray (ids 0xFFFFFFFF on a miss), ALIVE, the
 * successor state in the input layout (ALIVE only; its medium fields only when InMedium), the slot value after the bounce and the carried
 * RNG state (0 unless the path ended under B200PT_BQ_CARRY).  *survivors: the survivor count the kernels wrote.  Waits for the waves in
 * flight; the accumulation, the dispatch counter and the adaptive state are not touched; the work counters are.  Throughput, radiance, pdf,
 * medium and slot values may be anything.  B200PT_ERR_NO_SCENE without a scene, an environment map or the LUTs; B200PT_ERR_WRONG_ARGUMENTS
 * for volumes or the atmosphere, a non-finite origin, a zero or non-finite direction, Depth >= MaxDepth, DFLAGS bits 29-30 set or unknown
 * flag bits. */
#define B200PT_BQ_STORE       2
#define B200PT_BQ_CARRY       4
#define B200PT_BQ_IN_ORG      0    /* origin, then the pdf of the segment's BSDF sample */
#define B200PT_BQ_IN_PDF      3
#define B200PT_BQ_IN_DIR      4    /* direction, then the sampler state (u32 bits) */
#define B200PT_BQ_IN_RNG      7
#define B200PT_BQ_IN_THR      8    /* throughput, then DFLAGS (u32 bits) */
#define B200PT_BQ_IN_DFLAGS   11
#define B200PT_BQ_IN_RAD      12   /* radiance gathered so far, then the sample slot (u32 bits) */
#define B200PT_BQ_IN_SLOT     15
#define B200PT_BQ_IN_MEDIUM   16   /* medium colour, density */
#define B200PT_BQ_IN_MEDIUM_G 20   /* medium anisotropy */
#define B200PT_BQ_IN_SAMPLE   21   /* sample slot value before the bounce (4 floats) */
#define B200PT_BQ_IN_STRIDE   25
#define B200PT_BQ_OUT_T       0
#define B200PT_BQ_OUT_U       1
#define B200PT_BQ_OUT_V       2
#define B200PT_BQ_OUT_INST    3    /* u32 bits */
#define B200PT_BQ_OUT_PRIM    4    /* u32 bits */
#define B200PT_BQ_OUT_ALIVE   5
#define B200PT_BQ_OUT_NEXT    6    /* B200PT_BQ_IN_SAMPLE floats in the input layout */
#define B200PT_BQ_OUT_SAMPLE  27
#define B200PT_BQ_OUT_CARRY   31   /* u32 bits */
#define B200PT_BQ_OUT_STRIDE  32
int32_t b200pt_bounce_query(b200pt_handle h, uint32_t n, const float *in, uint32_t flags, float *out, uint32_t *survivors);

/* Energy-compensation lookup-table baker (SURVEY.md 8f row 2).
 * Replaces LookupTableCalculator::CalculateTable(tableSize, sampleCount) (PathTracer/LookupTableCalculator.h:8,
 * LookupTableCalculator.cpp:44-157) with its shaders LookupReflect.slang / LookupRefract.slang (ABOVE_SURFACE / BELOW_SURFACE).
 * kind: 0 = reflection {64,64,32}, 1 = refraction hit-from-outside {128,128,32}, 2 = refraction hit-from-inside {128,128,32}
 * (sizes as Application.cpp:41,54,67 passes them; any size is accepted).  out = sx*sy*sz floats, layout [z][y][x] as the .bin files.
 * sample_count is rounded down to a multiple of 20 like the reference (20 samples per dispatch).  `seed` replaces the wall-clock
 * term of the reference's per-dispatch seed, making a bake reproducible.  slices: 0 = auto; 1 = the reference's fp32 summation order.
 * elapsed_ms (optional): device time of the bake kernels (CUDA events). */
int32_t b200pt_bake_lut(b200pt_handle h, int32_t kind, uint32_t sx, uint32_t sy, uint32_t sz, uint32_t sample_count, uint32_t seed,
                        uint32_t slices, float *out, float *elapsed_ms);
/* Application.cpp:35-72: write ReflectionLookup.bin / RefractionLookupHitFromOutside.bin / RefractionLookupHitFromInside.bin into dir
 * (only the missing ones unless overwrite != 0); the reference uses sample_count = 10,000,000. */
int32_t b200pt_bake_luts_to_dir(b200pt_handle h, const char *dir, uint32_t sample_count, uint32_t seed, int32_t overwrite);
int32_t b200pt_scene_stats(b200pt_handle h, uint32_t *triangles, uint32_t *bvh_nodes, uint32_t *emissive_meshes, uint32_t *textures);

/* Host half of the acceleration-structure build (replaces the driver's BLAS/TLAS build behind VH/Source/Vulkan/BLASBuilderImpl.cpp,
 * TLASImpl.cpp for scenes that traverse out of L2): collapse of the GPU-built BVH2 into 128-byte BVH4 nodes.  Pure CPU code, exposed so
 * the structure can be checked without a GPU.  nodes2: n_nodes2 x 64-B {lo0[3],hi0[3],lo1[3],hi1[3],c0,c1,pad[2]} with child >= 0 an
 * inner node and child < 0 a leaf reference; nodes4_out: room for n_nodes2 x 128-B {lox[4],loy[4],loz[4],hix[4],hiy[4],hiz[4],child[4],pad[4]}.
 * Returns the node count in *n_nodes4_out (0 when root2 is a leaf) and the BVH4 depth in *depth_out. */
int32_t b200pt_bvh4_collapse(const void *nodes2, uint32_t n_nodes2, int32_t root2, void *nodes4_out, uint32_t *n_nodes4_out, int32_t *depth_out);

/* Opt-in tree-quality pass (B200PT_BVH_SAH=1 at SetScene time): binned-SAH rebuild of the inner nodes above the leaves of the GPU LBVH.
 * Pure CPU code, exposed for tests and offline experiments.  nodes2 / nodes_out: n_nodes2 x 64-B BVH2 nodes (layout as in
 * b200pt_bvh4_collapse); *n_out = leaves - 1 nodes written in depth-first order with root 0 (0 if nothing could be rebuilt);
 * sah_before_after[2]: surface-area-heuristic cost of the input and of the output, relative to the root box. */
int32_t b200pt_bvh2_sah_rebuild(const void *nodes2, uint32_t n_nodes2, int32_t root2, void *nodes_out, uint32_t *n_out, int32_t *depth_out, double *sah_before_after);

/* Second opt-in level (B200PT_BVH_SAH=2): binned-SAH build from the per-slot reference boxes; leaves of <= 4 references are re-formed.
 * ref_boxes: n x 6 floats (lo xyz, hi xyz); nodes_out: room for n - 1 nodes; perm_out[new slot] = old slot; trav_cost = price of a node
 * visit in triangle tests (1.0 = classic SAH).  *n_out = 0 when n <= 4 (one leaf) or a box is inverted / NaN. */
int32_t b200pt_bvh2_sah_build(const float *ref_boxes, uint32_t n, float trav_cost, void *nodes_out, uint32_t *perm_out, uint32_t *n_out, int32_t *depth_out, double *sah_cost);

/* Third opt-in level (B200PT_BVH_SAH=3 = level 2 followed by this): insertion-based refinement of a BVH2 -- the `fraction` largest nodes
 * are re-inserted where they add the least surface area, `passes` times.  Leaves are kept; output conventions as b200pt_bvh2_sah_rebuild. */
int32_t b200pt_bvh2_reinsert(const void *nodes2, uint32_t n_nodes2, int32_t root2, void *nodes_out, int32_t passes, float fraction, uint32_t *n_out, int32_t *depth_out, double *sah_before_after);

/* GPU tree builder (update_instance_transforms with B200PT_REBUILD_GPU): PLOC clustering over reference boxes in the given (Morton) order,
 * leaves of <= 4 references by the SAH leaf rule, nodes depth-first with root 0, perm_out[new slot] = old slot.  Pure CPU restatement of the
 * device builder, with the conventions of b200pt_bvh2_sah_build (trav_cost 1): *n_out = 0 when n <= 4 or a box is inverted / NaN. */
int32_t b200pt_bvh2_ploc_build(const float *ref_boxes, uint32_t n, void *nodes_out, uint32_t *perm_out, uint32_t *n_out, int32_t *depth_out, double *sah_cost);
/* Test hook: the device builder and the device BVH4 collapse the engine runs, on these boxes.  nodes_out: room for n - 1 BVH2 nodes,
 * perm_out: n entries, nodes4_out: room for n - 1 BVH4 nodes (layouts as in b200pt_bvh4_collapse).  Equals b200pt_bvh2_ploc_build and
 * b200pt_bvh4_collapse of its nodes bit for bit; rejects what b200pt_bvh2_ploc_build rejects (zero counts). */
int32_t b200pt_bvh2_ploc_build_query(b200pt_handle h, const float *ref_boxes, uint32_t n, void *nodes_out, uint32_t *perm_out, uint32_t *n_out, int32_t *depth_out,
                                     void *nodes4_out, uint32_t *n4_out, int32_t *depth4_out);

/* ---- standalone codecs of the loader / image-output API (no GPU needed) ---- */
/* stbi_load(.., STBI_rgb_alpha) / stbi_loadf semantics (AssetImporterImpl.cpp:494-545); free with b200pt_free */
int32_t b200pt_decode_image_file(const char *path, uint32_t *width, uint32_t *height, uint8_t **rgba_out);
int32_t b200pt_decode_hdr_file(const char *path, uint32_t *width, uint32_t *height, float **rgba_out);
int32_t b200pt_write_png(const char *path, uint32_t width, uint32_t height, const uint8_t *rgba);
/* host restatement of LoadEnvironmentMap's alias table (PathTracer.cpp:1137-1332); alias_out = width*height {u32,f32} */
int32_t b200pt_build_env_alias(float *rgba_inout, uint32_t width, uint32_t height, void *alias_out, float *sum_out);
/* parse a glTF into a heap-allocated scene description (b200pt_free_scene); what set_scene_file uploads */
int32_t b200pt_load_gltf(const char *path, b200pt_scene_desc **out);
int32_t b200pt_free_scene(b200pt_scene_desc *s);
void    b200pt_free(void *p);

#ifdef __cplusplus
}
#endif
#endif
