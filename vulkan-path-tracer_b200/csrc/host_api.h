// host_api.h -- host-side (C++17) pieces of the runtime above the C-ABI: codecs, glTF loader,
// environment-map preprocessing, camera, and the PathTracer / PostProcessor mirror classes.
#pragma once
#include "device_types.h"
#include <string>
#include <vector>
#include <memory>

namespace b200pt {

struct CudaError { int code; std::string what; };   // every failure crosses the C-ABI as a code + message (capi.cpp guard)

// ---- density_grid.cpp: AddDensityDataToVolume after the file read (PT/PathTracer.cpp:1391-1452) ----
struct PreparedGrid {
    std::vector<float> values, max_densities;       // temperature-patched values [z][y][x]; 32^3 majorants
    int imin[3], dim[3];
    float corner_min[3], corner_max[3], max_density;
    float wmin[3], wext[3], inv_vs[3], trans[3];    // SampleNanoVDBBuffer's per-grid constants (DevGrid)
    bool has_temperature = false;
};
void prepare_density_grid(const b200pt_density_grid &g, PreparedGrid &out);

// ---- image_codecs.cpp ----
bool decode_image_rgba8(const std::string &path, uint32_t &W, uint32_t &H, std::vector<uint8_t> &rgba, std::string &err);
bool decode_hdr_rgba32f(const std::string &path, uint32_t &W, uint32_t &H, std::vector<float> &rgba, std::string &err);
bool write_png_rgba8(const std::string &path, uint32_t W, uint32_t H, const uint8_t *rgba);

// ---- scene_loader.cpp : the loader's matrix arithmetic (float, row-major m[r][c]); animation.cpp poses with the same functions ----
struct M4 { float m[4][4]; };
M4 m4_identity();
M4 m4_mul(const M4 &a, const M4 &b);
void m4_to_colmajor(const M4 &a, float out[16]);
struct NodeTRS { bool has_matrix = false; M4 matrix; float t[3] = { 0, 0, 0 }, r[4] = { 0, 0, 0, 1 }, s[3] = { 1, 1, 1 }; };
M4 node_local(const NodeTRS &n);                    // matrix, or T * R * S

// ---- glTF animation data (scene_loader.cpp reads it, animation.cpp evaluates it).  Reading it never fails a load: a problem is kept in an
// err string and reported by the pose that needs the data.
struct AnimNode { NodeTRS trs; std::vector<int> children; int mesh = -1, skin = -1; bool has_weights = false; std::vector<float> weights; };
struct AnimSkin { std::vector<int> joints; std::vector<M4> inverse_bind; std::string err; };
enum AnimInterp { INTERP_STEP = 0, INTERP_LINEAR = 1, INTERP_CUBIC = 2 };
enum AnimPath { PATH_T = 0, PATH_R = 1, PATH_S = 2, PATH_W = 3 };
struct AnimSampler { std::vector<float> input, output; int interp = INTERP_LINEAR; uint32_t comps = 0; std::string err; };   // comps: output floats per key value
struct AnimChannel { int node = -1, path = PATH_T, sampler = -1; };
struct AnimClip { std::string name; std::vector<AnimSampler> samplers; std::vector<AnimChannel> channels; float t0 = 0.0f, t1 = 0.0f; std::string err; };
struct AnimPrim {                                   // one per HostMesh, i.e. per loaded glTF primitive
    int gltf_mesh = -1;
    uint32_t count = 0;                             // vertices
    uint32_t sets = 0;                              // JOINTS_n / WEIGHTS_n pairs
    std::vector<uint32_t> joints; std::vector<float> weights;   // [vertex][4 * sets]
    uint32_t targets = 0;                           // morph targets; dpos / dnrm / duv: [target][vertex][3 | 3 | 2], empty when no target has the attribute
    std::vector<float> dpos, dnrm, duv;
    std::vector<float> rest;                        // [vertex][8] position, NORMAL as stored (not normalised), uv; only for primitives with joints or targets
    bool gen_normals = false;                       // no NORMAL: the loader generated them (last face wins)
    std::vector<uint32_t> last_face;                // gen_normals: per vertex the last face that uses it (UINT32_MAX: none)
    std::string err;
};
struct HostAnimation {
    std::vector<AnimNode> nodes;
    std::vector<int> roots;                         // the loaded scene's root nodes
    std::vector<int> instance_node;                 // per HostScene instance: the node that produced it (loader DFS order)
    std::vector<std::vector<float>> mesh_weights;   // per glTF mesh: mesh.weights (empty: absent)
    std::vector<uint32_t> mesh_targets;             // per glTF mesh: morph target count of its primitives
    std::vector<AnimSkin> skins;
    std::vector<AnimPrim> prims;
    std::vector<AnimClip> clips;
    std::vector<int> deformable;                    // HostMesh indices some skin or morph target touches, ascending
    std::vector<int> prim_skin;                     // per HostMesh: the skin of the nodes that instance it (-1: none)
    std::string err;                                // node-graph problems
};

// ---- scene_loader.cpp : what AssetImporter::ImportScene + PathTracer::SetScene keep (Asset.h:131-138) ----
struct HostMesh { std::vector<b200pt_vertex> vertices; std::vector<uint32_t> indices; std::string name; };
struct HostTexture { uint32_t width = 0, height = 0, channels = 0; std::vector<uint8_t> data; };
struct HostScene {
    std::vector<HostMesh> meshes;
    std::vector<b200pt_material> materials;
    std::vector<std::string> material_names;
    std::vector<HostTexture> textures;
    std::vector<b200pt_instance> instances;
    float camera_view[16];
    float camera_aspect = 1.0f;
    std::shared_ptr<const HostAnimation> animation;  // glTF files only (nodes, skins, morph targets, animations); null for OBJ and arrays
};
bool load_gltf_scene(const std::string &path, HostScene &out, std::string &err);   // .gltf / .glb
bool load_obj_scene(const std::string &path, HostScene &out, std::string &err);    // .obj + .mtl (assimp semantics from upstream knowledge)
bool load_scene_file(const std::string &path, HostScene &out, std::string &err);   // by extension, like AssetImporter::ImportScene
bool scene_from_desc(const b200pt_scene_desc *d, HostScene &out, std::string &err);

// ---- animation.cpp : a pose of a loaded glTF scene at time t (glTF 2.0 Appendix C), on the host ----
struct HostPose {
    std::vector<M4> world;                          // per node: glTF world matrix (no flip)
    std::vector<std::vector<float>> weights;        // per node: morph weights of its mesh (empty: no mesh or no targets)
    std::vector<b200pt_instance> instances;         // the scene's instances with their posed transforms
    std::vector<float> palette;                     // per deformable mesh (HostAnimation::deformable order), joint matrices, 12 floats (3x4 row-major) each
    std::vector<uint32_t> palette_base;             // per deformable mesh: first joint in palette (joint count = palette_base[d + 1] - palette_base[d])
    std::vector<float> morph;                       // per deformable mesh, its target weights
    std::vector<uint32_t> morph_base;               // as palette_base, in floats
};
void finalize_animation(HostAnimation &a, const HostScene &sc);   // deformable / prim_skin, after the loader filled the rest
uint32_t animation_range(const AnimClip &c, float *t0, float *t1);   // returns the channel count; t0 / t1 of the valid samplers (0 when none)
// animation -1: the rest pose.  Throws CudaError{WRONG_ARGUMENTS} for malformed data the pose needs or a mesh its instances deform two ways.
void evaluate_pose(const HostAnimation &a, const HostScene &sc, int animation, float t, HostPose &out);

// ---- env_camera.cpp ----
// PathTracer::LoadEnvironmentMap (PathTracer.cpp:1137-1332): alias table + pdf in alpha. Returns the importance sum.
float build_env_alias(float *rgba, uint32_t width, uint32_t height, uint2 *alias_out);
// Editor/FlyCamera round trip (Editor.cpp:45-48,1042-1051; FlyCamera.cpp:84-140)
void camera_from_view(const float view[16], float aspect, float viewInv[16], float projInv[16]);
void mat3_inverse_from_o2w(const float o2w[12], float w2o[9]);

// ---- bloom mip chain sizes (PostProcessor.cpp:128-158) ----
uint32_t bloom_mip_sizes(uint32_t W, uint32_t H, uint32_t wh[20]);

// partition helpers
uint32_t partition_global_row(uint32_t local_row, uint32_t rank, uint32_t world, uint32_t band);
uint32_t partition_local_rows(uint32_t H, uint32_t rank, uint32_t world, uint32_t band);

} // namespace b200pt
