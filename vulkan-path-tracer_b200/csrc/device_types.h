// device_types.h -- POD layouts shared by the host runtime and the sm_90a kernels.
// HBM layout of the scene (all read-only during rendering, replicated per GPU):
//   vertices  : b200pt_vertex[ ]   32 B, all meshes concatenated          (SH/Bindings.slang:7-12)
//   indices   : u32[ ]             all meshes concatenated, mesh-local    (PT/PathTracer.cpp:216)
//   meshes    : DevMesh[ ]         {vertex base, index base, triangles}
//   instances : DevInstance[ ]     object->world 3x4, world->object 3x3, mesh, material (TLAS instance order)
//   materials : b200pt_material[ ] 112 B                                  (PT/PathTracer.h:12-34)
//   textures  : DevTexture[ ]      RGBA8 / R8 texel arrays                (PT/PathTracer.cpp:812-869)
//   emissive  : DevEmissive[ ]     80 B                                   (PT/PathTracer.h:321-328)
//   env       : float4[W*H] (rgb, pdf) + alias uint2[W*H]                 (PT/PathTracer.cpp:1137-1332)
//   luts      : float[32*64*64], float[32*128*128] x2                     (PT/PathTracer.cpp:199-201)
//   bvh       : BvhNode[ ] 64 B (two child boxes per node) + BvhTri[ ] 48 B (v0,e1,e2 + ids), Morton order
#pragma once
#include <stdint.h>
#include "../../include/b200pt.h"

#include <cuda_runtime.h>

namespace b200pt {

struct DevMesh { uint32_t vbase, ibase, tri_count, _pad; };

struct DevInstance {
    float o2w[12];      // row-major 3x4
    float w2o[9];       // row-major 3x3 inverse of the linear part
    uint32_t mesh, material, tri_base;
    uint32_t emissive_tri_count;   // TriangleCount of this instance's EmissiveMeshEntry, 0 if not emissive
    uint32_t _pad[3];
};                      // 112 B
static_assert(sizeof(DevInstance) == 112, "DevInstance layout");

struct DevTexture { const uint8_t *data; uint32_t w, h, c, _pad; };

// Reference material (112 B, PT/PathTracer.h:12-34) + the texel values of its 1x1 textures resolved on the host:
// the default white / (128,128,255) textures (PT/PathTracer.cpp:1557-1621) then cost no dependent texture fetch at all.
struct DevMaterial {
    b200pt_material m;
    uint32_t const_mask;     // bit0 base colour, bit1 normal, bit2 roughness, bit3 metallic, bit4 emissive: that texture is 1x1
                             // bit5: pre0..pre3 below are valid (bits 0,2,3,4 all set: nothing of the material depends on the hit's uv)
    float crough, cmetal;    // R channel / 255
    uint32_t _pad;
    float4 cbase, cnormal, cemis;   // RGBA / 255
    // uv-independent part of Material construction (SH/Material.slang:39-77) and of the lobe probabilities (:169-177), evaluated
    // ONCE per material by k_prepare_materials (wavefront_kernels.cu) with the very device functions the per-hit path uses
    float4 pre0;             // BaseColor * texel^2.2 (rgb) | Roughness * texel
    float4 pre1;             // EmissiveColor * texel (rgb) | Metallic * texel
    float4 pre2;             // Ax | Ay | max(IOR, 1.000001) | 0
    float4 pre3;             // pm | pd | pg | 0
};
static_assert(sizeof(DevMaterial) == 240, "DevMaterial layout");

struct DevEmissive { uint32_t mesh, material, tri_count, instance; float xf[16]; };  // PT/PathTracer.h:321-328 (80 B)
static_assert(sizeof(DevEmissive) == 80, "EmissiveMeshEntry is 80 B");
static_assert(sizeof(b200pt_vertex) == 32, "Vertex is 32 B");
static_assert(sizeof(b200pt_material) == 112, "Material is 112 B");

// 64-byte BVH2 node: AABBs of both children live in the parent, so one 64-B fetch decides both.
// child >= 0 : internal node index;  child < 0 : leaf, r = ~child, first Morton slot = r >> 2, triangle count = (r & 3) + 1
struct BvhNode {
    float lo0[3], hi0[3];
    float lo1[3], hi1[3];
    int32_t c0, c1;
    uint32_t _pad[2];
};
static_assert(sizeof(BvhNode) == 64, "BvhNode is 64 B");

// 128-byte BVH4 node (wide traversal of scenes that live in L2/HBM): the four child boxes in SoA order, so a node is eight 16-B loads and
// one memory round trip decides four children.  Built on the host by collapsing the GPU-built BVH2 (lbvh.cu: bvh4_collapse_host).
// child >= 0 : BVH4 node index;  child < 0 : leaf reference, same encoding as BvhNode;  unused slot: child = BVH4_EMPTY and a point box
// at +3e38 that no ray interval reaches (no special case in the traversal).
struct Bvh4Node {
    float lox[4], loy[4], loz[4], hix[4], hiy[4], hiz[4];
    int32_t child[4];
    uint32_t _pad[4];
};
static_assert(sizeof(Bvh4Node) == 128, "Bvh4Node is 128 B");
constexpr int32_t BVH4_EMPTY = (int32_t)0x80000000;

// 48-byte triangle: world-space v0 and edges + ids (a = v0.xyz|gid, b = e1.xyz|inst, c = e2.xyz|prim)
struct BvhTri { float4 a, b, c; };
static_assert(sizeof(BvhTri) == 48, "BvhTri is 48 B");

// 112-byte per-triangle shading record, indexed by the global triangle id ((instance, primitive) order): one gather replaces the reference's
// instance -> mesh -> index -> vertex descriptor chain (SH/ClosestHit.slang:46-57, SH/Surface.slang:33-41).
//   r0 = P1.xyz | instance   r1 = P2.xyz | primitive   r2 = P3.xyz | material
//   r3 = N1.xyz | uv1.x      r4 = N2.xyz | uv1.y       r5 = N3.xyz | uv2.x      r6 = uv2.y uv3.x uv3.y 0   (object space)
struct ShadeTri { float4 r[7]; };
static_assert(sizeof(ShadeTri) == 112, "ShadeTri is 112 B");

// 64-byte emissive triangle: world-space corners (EmissiveMeshEntry::Transform applied, SH/Sampler.slang:389-391) + uvs
//   r0 = p0.xyz | uv0.x   r1 = p1.xyz | uv0.y   r2 = p2.xyz | uv1.x   r3 = uv1.y uv2.x uv2.y | global triangle id (bits)
struct EmTri { float4 r[4]; };

// 128-byte volume (VolumeGPU of PT/PathTracer.h:341-395): mn_density = CornerMin | Density, mx_g = CornerMax | Anisotropy, color_alpha = Color | Alpha,
// emis_droplet = EmissiveColor | DropletSize, flags = { ApproximatedScattering, HasTemperatureData, UseBlackbody, grid slot (0xFFFFFFFF: homogeneous) },
// tcol_gamma = TemperatureColor | TemperatureGamma, tparams = { TemperatureScale, EmissiveColorGamma, ApproximatedScatteringFalloff, GridSharpness },
// kelvin = { (float)KelvinMin, (float)(KelvinMax - KelvinMin), MaxDensityInTheGrid, - }
struct DevVolume { float4 mn_density, mx_g, color_alpha, emis_droplet; uint4 flags; float4 tcol_gamma, tparams, kelvin; };
static_assert(sizeof(DevVolume) == 128, "DevVolume is 128 B");
// Density data of one heterogeneous volume (PT/PathTracer.cpp:1346-1516): a dense copy of the values the reference keeps in a NanoVDB buffer, the
// 32^3 majorants, and the constants SampleNanoVDBBuffer (SH/Volume.slang:69-117) derives from the grid header on every call.
struct DevGrid {
    const float *values;       // [z][y][x] over the active-voxel bbox
    const float *max_densities; // 32768
    int imin[3]; int dim[3];   // root bbox: imin .. imin + dim - 1
    float wmin[3], wext[3];    // (float)floor(world bbox min), (float)(ceil(world bbox max) - floor(world bbox min))
    float inv_vs[3], trans[3]; // NanoVDB Map: mInvMatF diagonal, mVecF
};

struct DevScene {
    const b200pt_vertex *verts;
    const uint32_t *indices;
    const DevMesh *meshes;
    const DevInstance *instances;
    const DevMaterial *materials;
    const DevTexture *textures;
    const DevEmissive *emissive;
    const float4 *env;
    const uint2 *alias;
    const float2 *env_row_cos;     // per env-map row py: { cos(py*stepTheta), cos(py*stepTheta + stepTheta) } (SH/Sampler.slang:329-331), host-evaluated
    const float *lut_reflect, *lut_refract_out, *lut_refract_in;
    const uint32_t *tri_slot;      // global triangle id -> one of its BvhTri slots (light-ray visibility test in k_connect)
    const uint8_t *tri_class;      // global triangle id -> shading class of its material (MaterialClass): selects the hit queue / k_shade_hit instantiation
    const BvhNode *nodes;
    const Bvh4Node *nodes4;        // BVH4 collapse of `nodes` (nullptr when the scene is traversed as BVH2), root = node 0
    const BvhTri *tris;
    const ShadeTri *shade_tris;
    const EmTri *em_tris;
    const uint32_t *em_tri_base;   // per emissive mesh: first EmTri
    const DevVolume *volumes;      // AABB volumes (volumes.cuh), n_volumes entries
    const DevGrid *grids;          // density data of the heterogeneous ones (DevVolume::flags.w)
    uint32_t n_grids;              // != 0: NEE transmittance is a random walk on the path's stream and moves from the shading kernels into k_connect
    uint32_t uniform_class;        // the one MaterialClass every triangle has, or 0xFF (k_extend then looks tri_class up per hit)
    uint32_t pre_pass;             // k_volume_decide runs before k_extend (the scene has volumes or the atmosphere is on): hit records may hold VOLUME_EVENT / DEAD_EVENT
    uint32_t n_volumes, phase_function;   // phase_function: 0 HG, 1 Draine, 2 HG + Draine (PT/PathTracer.h:76-81)
    uint32_t n_emissive, envW, envH, n_tris, n_nodes, n_nodes4;
    int32_t root;            // child-style reference of the root
    uint32_t bvh_bytes;      // nodes+tris size if they are contiguous and small enough to stage in smem, else 0
    uint32_t n_flat;         // != 0: the scene has so few triangle slots that shared-memory traversals test them all in order, no hierarchy (bvh_traverse.cuh)
};

// Shading classes = the lobe sets of SH/Material.slang:169-177 that a material can ever sample or evaluate.  The lobe probabilities are
// pm = Metallic, pd = (1-Metallic)(1-Transmission), pg = (1-Metallic)Transmission (normalised); when the metallic texture is 1x1 they are
// per-material constants, and for the three pure cases two of them are EXACTLY 0, so the corresponding lobe code contributes exact zeros and
// can be compiled out of that class's kernel (k_shade_hit<CLASS>).  k_extend sorts hits into one queue per class (material-sorted shading).
enum MaterialClass : uint32_t { MC_DIFFUSE = 0,   // Metallic*texel == 0 and Transmission == 0: diffuse + dielectric specular
                                MC_METAL = 1,     // Metallic*texel == 1: metallic lobe only
                                MC_GLASS = 2,     // Metallic*texel == 0 and Transmission == 1: glass reflect + refract
                                MC_GENERAL = 3,   // anything else (mixed lobes, textured metallic)
                                MC_COUNT = 4 };
// Control block (u32 words): [0],[1] live-path counts by bounce parity p; [8+p] / [10+p] fetch counters of k_extend_dyn / k_shadow_dyn;
// [CTRL_Q + 8p + 0] miss-queue length, [CTRL_Q + 8p + 1 + c] hit-queue length of class c for a bounce of parity p.
constexpr uint32_t CTRL_Q = 16u, CTRL_WORDS = 32u;
constexpr uint32_t Q_NONE = 7u;   // queue code of an inactive lane
// The hit / miss queues of one bounce: entries are indices into the dense PathState arrays.  Class c owns hit[c * cap .. c * cap + count_c).
struct Queues { uint32_t *miss; uint32_t *hit; uint32_t cap; };

struct DevConfig {          // PT/PathTracer.h:271-302 (the fields the surface integrator reads)
    float VI[16], PI[16];
    uint32_t SampleCount, MaxDepth;
    float MaxLuminance, FocusDistance, DepthOfFieldStrength;
    float SkyRotationAzimuth, SkyRotationAltitude, EnvironmentIntensity, EmissiveMeshSamplingPDFBias;
    uint32_t ScreenSplitCount;
    uint32_t EnableSkyMIS, EnableMeshMIS, ShowEnvMapDirectly, UseOnlyGeometryNormals, UseEnergyCompensation, FurnaceTestMode;
    uint32_t W, H;           // full image size
    uint32_t rank, world, band_rows, local_rows;
    float cosAz, sinAz, cosAl, sinAl;   // cos/sin(SkyRotation{Azimuth,Altitude} / 180 * PI), evaluated on the host
    // atmosphere (ENABLE_ATMOSPHERE + SH/Bindings.slang:26-37; csrc/atmosphere.cuh)
    uint32_t EnableAtmosphere;
    float PlanetPosition[3], PlanetRadius, AtmosphereHeight;
    float RayleighMult[3], MieMult[3], OzoneMult[3];
    float RayleighDensityFalloff, MieDensityFalloff, OzoneDensityFalloff, OzonePeak;
    float SunColor[3];
    float cosSunTheta;       // cos(0.004675), SH/Sampler.slang:469 (host-evaluated)
};

struct DevDispatch { uint32_t FrameCount, Seed, ChunkIndex, _pad; };   // PT/PathTracer.h:304-309

// ---- wavefront SoA (all float4 so every access is a coalesced 16-B lane access) ----
struct PathState {
    float4 *org_pdf;     // Origin.xyz, PDF of the previous BSDF sample (payload.PDF)
    float4 *dir_rng;     // Direction.xyz, RNG state (u32 bits)
    float4 *thr_depth;   // pathThroughput.xyz, Depth | InMedium<<31 (u32 bits)
    float4 *rad_slot;    // pathLight.xyz, sample slot (u32 bits)
    float4 *medium;      // MediumColor.xyz, MediumDensity
    float  *medium_g;    // MediumAnisotropy
    uint32_t *vol_depth; // payload.VolumeDepth (nullptr while the scene has no volumes)
};
struct ShadeOut {
    float4 *hit;         // t, u, v, tri slot (u32 bits; 0xFFFFFFFF = miss)
    float4 *bxdf_pdf;    // payload.BxDF.xyz, payload.PDF
    float4 *e0;          // emission term of payload.Emitted (xyz), new Depth (u32 bits)
    float4 *sky_o, *sky_d, *sky_c;   // shadow ray origin(w: valid), direction, weighted contribution
    float4 *lit_o, *lit_d, *lit_c;   // lit_o.w: valid, lit_d.w: expected prim (bits), lit_c.w: expected inst (bits)
};

struct WaveCounters {    // device-side counters (u64)
    unsigned long long paths, extend_rays, shade_invocations, surface_hits, misses, shadow_rays, medium_events;
};

} // namespace b200pt
