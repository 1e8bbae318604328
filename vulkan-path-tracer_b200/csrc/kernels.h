// kernels.h -- host-callable launchers of the sm_90a kernels (wavefront_kernels.cu, lbvh.cu, post_kernels.cu, denoise_kernels.cu, trace_query.cu)
#pragma once
#include "device_types.h"
#include "cuda_resources.h"
#include <cuda_runtime.h>
#include <vector>

namespace b200pt {

struct LaunchCfg {
    int grid_light;     // grid for streaming kernels (raygen / resolve / post)
    int grid_volume_decide;   // persistent grid of k_volume_decide (256 threads per CTA)
    int grid_extend, grid_connect;   // persistent grids of the traversal kernels (SM count x resident CTAs of each kernel)
    int grid_shade;     // persistent grid for the shading kernel
    int max_stack;      // traversal stack entries (BVH depth + 2)
    bool bvh_in_smem;   // whole BVH staged to shared memory by TMA
    bool trav_dyn;      // dynamic-fetch while-while traversal kernels (k_extend_dyn / k_shadow_dyn) instead of one ray per thread
    int dyn_thresh;     // a warp refills its idle lanes when fewer than this many lanes are still traversing
    int grid_shadow;    // persistent grid of k_shadow_dyn
    bool wide;          // the dynamic-fetch kernels walk the BVH4 (DevScene::nodes4)
    int dyn_stack;      // shared-memory stack entries per thread of the dynamic-fetch kernels (BVH4: overflow goes to local memory)
    int wide_cap;       // BVH4: most shared-memory stack entries per thread (B200PT_WIDE_STACK, default WIDE_STACK_DEFAULT)
    bool big;           // bvh_in_smem with a BVH > 64 KiB: one 512-thread CTA per SM for k_extend, k_camera, k_connect and the fused k_shade_hit
    int extend_threads; // CTA size of k_extend / k_extend_dyn, k_camera and k_connect (256; big mode's one-ray-per-thread kernels: 512)
    int bounce_threads; // CTA size of the fused k_shade_hit (128, big: 512)
    int fuse;           // 0: k_shade_hit + k_connect; 1: NEE queries + path epilogue inside k_shade_hit (no k_connect)
    int grid_bounce;    // persistent grid of the fused k_shade_hit (BVH + stacks in shared memory)
    bool camera;        // camera rays generated and traced by k_camera (shared-memory BVH, one ray per thread) when the call has no pre-pass
    int grid_camera;    // persistent grid of k_camera (extend_threads per CTA)
    int grid_features;  // persistent grid of k_features (256 threads per CTA)
    // dynamic shared memory (traversal stacks + the staged BVH) of each launch shape
    size_t smem_extend; // k_extend / k_extend_dyn, k_camera and the tracing k_connect (extend_threads per CTA)
    size_t smem_shadow; // k_shadow_dyn (256 threads, + its ray ring)
    size_t smem_bounce; // fused k_shade_hit (bounce_threads)
    size_t smem_trace;  // k_volume_decide and k_features (256 threads)
};

// Grids, CTA sizes and shared memory of every traversal launch for one scene, and the per-device shared-memory opt-in of every kernel the
// launchers can choose.  Runs on the engine's device before its first launch.
int query_launch_cfg(const DevScene &sc, int bvh_max_depth, int bvh4_depth, LaunchCfg *lc);
// The choices of one Engine::path_trace call (plan_call), passed to the launchers.
struct CallPlan {
    bool pre;           // k_volume_decide + k_shade_volume run (volumes or atmosphere): DevScene::pre_pass
    bool fuse;          // LaunchCfg::fuse without a pre-pass: no launch_connect
    bool camera;        // LaunchCfg::camera without a pre-pass: launch_camera instead of launch_raygen + bounce 0's launch_extend
    bool uniform;       // k_extend / k_camera skip the per-hit class lookup: one material class, no pre-pass
    bool walks;         // k_connect<., ., true>: NEE transmittance walks (atmosphere or grid volumes)
    uint32_t class_mask;   // k_shade_hit<CLASS> runs for every set bit
    bool implied;       // bounce 0 may run with WAVE_IMPLIED
    bool store;         // sub-wave 0 may run with WAVE_STORE
};
CallPlan plan_call(const LaunchCfg &lc, const DevScene &sc, const DevConfig &cfg, bool medium, uint32_t class_mask);
// ---- per-launch flags of the ray-generation and shading launchers (Engine::path_trace sets them per sub-wave and bounce) ----
// WAVE_IMPLIED: k_camera ran with ScreenSplitCount == 1 in a fused pipeline, so every camera path is inside the image.  k_camera writes
//               only dir_rng, the hit record and the queue entry; bounce 0's k_shade_miss and fused k_shade_hit take throughput, depth,
//               radiance, slot and pdf from camera_implied_* instead of loading them (the origin is not read at depth 0 outside a medium).
// WAVE_STORE:   first sub-wave of a call without pre-pass or medium walks: every path ends exactly once, in a slot nothing else writes, so
//               a path end stores its radiance instead of adding it to the slot, and ray generation does not clear the slot.
// WAVE_CARRY:   another sub-wave of the same frames follows: path ends store their RNG state to rng_carry for it.
constexpr uint32_t WAVE_IMPLIED = 1u, WAVE_STORE = 2u, WAVE_CARRY = 4u;
// The launchers below return the number of kernels they enqueued.
// active (adaptive sampling): P is the active count and wave entry i of a dispatch traces local pixel active[i]; nullptr = every pixel
int launch_raygen(const LaunchCfg &lc, const DevConfig &cfg, const DevDispatch *disp, uint32_t n_disp, uint32_t P, uint32_t first_sample, uint32_t flags,
                  const uint32_t *rng_carry, PathState ps, float4 *sample_buf, uint32_t *ctrl, WaveCounters *ctr, cudaStream_t st, const uint32_t *active = nullptr);
// launch_raygen + the camera rays' launch_extend in one kernel (CallPlan::camera): writes the path state, the hit records (hit_out) and the
// parity-0 queues.  The control block must be zero when it starts.
int launch_camera(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, const DevConfig &cfg, const DevDispatch *disp, uint32_t n_disp, uint32_t P,
                  uint32_t first_sample, uint32_t flags, const uint32_t *rng_carry, PathState ps, float4 *sample_buf, float4 *hit_out, uint32_t *ctrl, Queues q,
                  WaveCounters *ctr, cudaStream_t st, const uint32_t *active = nullptr);
// ---- adaptive sampling: per local pixel one 16-B record {meanL, M2 (float bits), n_p, flags} (Engine::d_px_state_) ----
constexpr uint32_t ADAPTIVE_TILE = 2048;      // pixels per block of the two compaction passes
constexpr uint32_t PX_CONVERGED = 1u;         // flags bit: the pixel is never traced again
// k_resolve over the active list: folds slot b * A + i of every dispatch into pixel active[i] with the pixel's own count, updates its record
void launch_resolve_adaptive(const LaunchCfg &lc, const DevConfig &cfg, uint32_t n_disp, uint32_t A, const uint32_t *active,
                             const float4 *sample_buf, float4 *image, uint4 *state, cudaStream_t st);
// decision at an interval boundary (decide: flag the converged pixels; otherwise only rebuild the list), then the stable compaction of the
// active pixels into `active` and their count into *active_count (device).  tile_count: ceil(npix / ADAPTIVE_TILE) words of scratch.
void launch_adaptive_update(uint4 *state, uint32_t npix, float threshold, uint32_t min_samples, bool decide, uint32_t *tile_count,
                            uint32_t *active, uint32_t *active_count, cudaStream_t st);
// ---- denoiser (denoise_kernels.cu) ----
constexpr float DN_UNKNOWN_VARIANCE = 1e30f;  // variance of a pixel with fewer than two frames
using FeaturesKernel = void (*)(DevScene, DevConfig, float3, uint32_t, uint32_t, int, float4 *, float4 *);
FeaturesKernel features_kernel(bool smem);   // k_features<smem>
// k_features over the local rows: albedo_cov = (mean albedo, hit fraction), normal_depth = (mean shading normal, mean view depth of the hits).
// forward: unit view direction of the image centre; seed0 = PCG_HASH(0x46454154).  Returns cudaError_t as int.
int launch_features(const LaunchCfg &lc, const DevScene &sc, const DevConfig &cfg, float3 forward, uint32_t samples, uint32_t seed0,
                    float4 *albedo_cov, float4 *normal_depth, cudaStream_t st);
void launch_record_variance(const uint4 *state, uint32_t npix, float *variance, cudaStream_t st);   // M2 / (n - 1) / n per record
// the a-trous filter on a W x H image (device buffers); scratch: 3 * W * H float4.  iterations == 0 copies color to out.
void launch_denoise_filter(uint32_t W, uint32_t H, const float4 *color, const float4 *albedo_cov, const float4 *normal_depth, const float *variance,
                           uint32_t iterations, float sigma_l, float sigma_n, float sigma_z, float4 *scratch, float4 *out, cudaStream_t st);
int launch_extend(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, PathState ps, float4 *hit_out, uint32_t *ctrl, uint32_t parity, Queues q,
                  WaveCounters *ctr, bool primary, cudaStream_t st);
// k_shade_miss + k_shade_hit<CLASS> for every class in cp.class_mask (+ k_shade_volume).
// cp.fuse: the bounce is finished inside k_shade_hit (the survivors are written compacted to dst), launch_connect is not called.
int launch_shade(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, const DevConfig &cfg, PathState ps, PathState dst, ShadeOut so, const float4 *hit_in,
                 uint32_t *ctrl, uint32_t parity, Queues q, float4 *sample_buf, uint32_t *rng_carry, WaveCounters *ctr, uint32_t flags, cudaStream_t st);
int launch_volume_decide(const LaunchCfg &lc, const DevScene &sc, const DevConfig &cfg, PathState ps, ShadeOut so, const uint32_t *ctrl, uint32_t parity,
                         float4 *sample_buf, uint32_t *rng_carry, cudaStream_t st);   // before launch_extend when the call has a pre-pass (CallPlan::pre)
int launch_connect(const LaunchCfg &lc, const CallPlan &cp, const DevScene &sc, const DevConfig &cfg, PathState src, PathState dst, ShadeOut so,
                   uint32_t *ctrl, uint32_t parity, Queues q, float4 *sample_buf, uint32_t *rng_carry, WaveCounters *ctr, uint32_t flags, cudaStream_t st);
void launch_resolve(const LaunchCfg &lc, const DevConfig &cfg, const DevDispatch *disp, uint32_t n_disp, uint32_t P,
                    const float4 *sample_buf, float4 *image, cudaStream_t st);
void launch_volume_walks(const DevScene &sc, uint32_t n, const float *org, const float *dir, const uint32_t *seeds, float ray_depth,
                         float *T_out, float *scatter_out, int32_t *vol_out, uint32_t *rng_out, cudaStream_t st);
// Shared-memory stack entries of the BVH4 dynamic-fetch kernels for a BVH4 of the given depth with a shared column of at most `cap` entries
// (the rest goes to the DYN_SPILL overflow array); 0 when even that cannot hold three pushes per level.
constexpr int WIDE_STACK_DEFAULT = 24;
int bvh4_stack_entries(int bvh4_depth, int cap);

// ---- traversal test hook (trace_query.cu, b200pt_trace_query): shapes and query kinds as in include/b200pt.h ----
enum { TQ_SHARED = 0, TQ_GLOBAL, TQ_FLAT, TQ_FIXED_ORIGIN, TQ_DYN2, TQ_DYN4, TQ_DYN4_SPILL, TQ_SHAPES };
enum { TQ_CLOSEST = 0, TQ_ANY, TQ_TARGET };
constexpr int TQ_UNSUPPORTED = -1;            // the scene has no such shape (no flat walk, no BVH4, too big for shared memory)
struct TraceQuery {                           // device arrays of n rays; target / tmax_test for TQ_TARGET, occluded for the any-hit kinds
    uint32_t n; const float *org, *dir, *tmin, *tmax, *tmax_test; const uint32_t *target;
    float *t; uint32_t *prim, *inst; float *uv; uint32_t *occluded; uint32_t *stats;   // stats: 3 per ray, or nullptr
};
// Returns cudaError_t as int, or TQ_UNSUPPORTED.
int launch_trace_query(const LaunchCfg &lc, const DevScene &sc, int bvh4_depth, int shape, int kind, bool fma, const TraceQuery &q, cudaStream_t st);

// ---- shading test hook (shade_query.cu, b200pt_shade_query) ----
struct ShadeQuery {                           // device arrays of n hits; L may be nullptr; out: n x B200PT_SQ_STRIDE floats
    uint32_t n; bool force_general; const uint32_t *gid, *rng; const float *uv, *dir, *org, *pay_pdf, *L; float *out;
};
int launch_shade_query(const DevScene &sc, const DevConfig &cfg, const ShadeQuery &q, cudaStream_t st);   // cudaError_t as int
struct MissQuery {                            // device arrays of n misses; out: n x B200PT_MQ_STRIDE floats (b200pt_miss_query)
    uint32_t n; const float *dir; const uint32_t *depth; const float *pay_pdf; float *out;
};
int launch_miss_query(const DevScene &sc, const DevConfig &cfg, const MissQuery &q, cudaStream_t st);     // cudaError_t as int

// ---- LBVH build (lbvh.cu): world-space flattening of the two-level TLAS/BLAS ----
// What lbvh_refit needs of a tree (per-slot slab assignment, BVH2 levels, BVH4 source map), derived at the first refit of that tree.
struct LbvhRefit { DevPtr<uint32_t> slot_jk; DevPtr<float> slot_box, node_box, bounds; DevPtr<int32_t> order, src4;
                   std::vector<uint32_t> level_off; uint32_t n4 = 0; bool ready = false; };
// One acceleration structure with its device blocks and its refit state: replacing or clearing a tree releases both.  nodes owns the one
// [nodes | tris] block; tris points into it, so it stays valid when the result is moved.  Move-only.
struct LbvhResult { DevPtr<ShadeTri> shade; DevPtr<uint32_t> tri_slot; DevPtr<BvhNode> nodes; BvhTri *tris; uint32_t n_nodes, n_tris; int32_t root; int max_depth; size_t bytes;
                    DevPtr<Bvh4Node> nodes4; uint32_t n_nodes4; int depth4;
                    uint32_t n_prims;                                        // triangle count
                    LbvhRefit refit; };
// Builds into ONE contiguous allocation [nodes | tris] (so small scenes can be staged to smem with one bulk copy).  The Morton-ordered
// per-slot reference boxes (n_tris x 6 floats) are handed out when asked for: host_ref_box receives a host copy (lbvh_refine_sah modes 2, 3),
// dev_ref_box the device array (lbvh_ploc_rebuild).  Returns cudaError_t as int.
int lbvh_build(const b200pt_vertex *d_verts, const uint32_t *d_indices, const DevMesh *d_meshes, const DevInstance *d_instances,
               uint32_t n_instances, uint32_t n_tris, LbvhResult *out, cudaStream_t st, std::vector<float> *host_ref_box = nullptr,
               DevPtr<float> *dev_ref_box = nullptr);
// BVH2 -> BVH4 on the host (pure CPU code, unit-tested without a GPU through b200pt_bvh4_collapse).  `out` must hold n_nodes2 entries.
// Returns the number of BVH4 nodes written (0 if the root is a leaf), *depth4 = depth of the BVH4 (root = 1).
uint32_t bvh4_collapse_host(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, Bvh4Node *out, int *depth4);
// Opt-in binned-SAH rebuild of the inner nodes above the LBVH's leaves (pure CPU code, unit-tested through b200pt_bvh2_sah_rebuild).
// `out` must hold n_nodes2 entries; returns the node count (0 = nothing rebuilt), *depth, sah[0/1] = SAH cost before / after.
uint32_t bvh2_sah_rebuild_host(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, BvhNode *out, int *depth, double sah[2]);
// Insertion-based refinement of any BVH2 (leaves kept); same output conventions as bvh2_sah_rebuild_host.
uint32_t bvh2_reinsert_host(const BvhNode *nodes2, uint32_t n_nodes2, int32_t root2, BvhNode *out, int passes, float fraction, int *depth, double sah[2]);
// Full binned-SAH build from per-slot reference boxes (n x 6 floats); leaves are re-formed, perm[new slot] = old slot; see lbvh.cu.
uint32_t bvh2_sah_build_host(const float *ref_boxes, uint32_t n, float trav_cost, BvhNode *out, uint32_t *perm, int *depth, double *sah_cost);
// PLOC build from reference boxes in Morton order (pure CPU code; the host restatement of ploc_build, which must match it bit for bit).
// Conventions and rejections of bvh2_sah_build_host; *depth = inner-node depth (root = 1).
uint32_t bvh2_ploc_build_host(const float *ref_boxes, uint32_t n, BvhNode *out, uint32_t *perm, int *depth, double *sah_cost);
// ---- GPU tree build (ploc.cu) ----
// The PLOC build of n reference boxes (device, Morton order, unpadded) into out (room for n - 1 nodes) and perm (n entries) on the device:
// *n_out nodes (0 when n <= LBVH_LEAF_MAX), *depth; the two come back in one readback.  h_small: caller-owned pinned host memory of 4 words
// for the readbacks (one per clustering step).  Returns cudaError_t as int.
int ploc_build(const float *d_ref_box, uint32_t n, BvhNode *d_out, uint32_t *d_perm, uint32_t *n_out, int *depth, uint32_t *h_small, cudaStream_t st);
// BVH2 -> BVH4 on the device, byte for byte bvh4_collapse_host's output (breadth-first, level by level).  d_out: room for n_nodes2 nodes.
// h_small: pinned host word for the per-level count.
int bvh4_collapse_device(const BvhNode *d_nodes2, uint32_t n_nodes2, int32_t root2, Bvh4Node *d_out, uint32_t *n4, int *depth4, uint32_t *h_small, cudaStream_t st);
// The GPU rebuild of an LBVH (update_instance_transforms(rebuild == 2)): ploc_build over the Morton-ordered reference boxes lbvh_build kept on the
// device, then the BvhTri slots permuted and tri_slot re-derived on the device.  A tree deeper than BVH_STACK_MAX - 2 and than the LBVH is
// dropped (the LBVH stays).  Returns cudaError_t as int.
int lbvh_ploc_rebuild(LbvhResult *r, DevPtr<float> ref_box, uint32_t *h_small, cudaStream_t st);
// lbvh_build_wide with the collapse on the device (scratch of n_nodes BVH4 nodes; r->nodes4 is allocated at the exact size).
int lbvh_build_wide_device(LbvhResult *r, uint32_t *h_small, cudaStream_t st);
// mode 1: inner nodes only (download, rebuild, upload in place); mode 2: full build from ref_box (the host reference boxes of lbvh_build),
// reference slots and tri_slot permuted (falls back to mode 1 when ref_box is null); mode 3: mode 2 + insertion-based refinement; 4: mode 1 +
// refinement; 5: refinement only.  Returns cudaError_t as int.
// A pass result deeper than BVH_STACK_MAX - 2 is dropped unless the input tree is deeper still (query_launch_cfg sizes the stacks from the depth).
constexpr int BVH_STACK_MAX = 64;
int lbvh_refine_sah(LbvhResult *r, const float *ref_box, cudaStream_t st, double sah[2], int mode = 1);
// Downloads r->nodes, collapses, uploads r->nodes4 (own allocation).  Returns cudaError_t as int; leaves nodes4 = nullptr if the root is a leaf.
int lbvh_build_wide(LbvhResult *r, cudaStream_t st);
// Refit in place after the instance transforms changed (d_instances holds the new o2w): the topology, slot order and tri_slot of r stay,
// every slot record and box, every reachable BVH2 child box (padded from the new scene bounds) and every BVH4 child box are recomputed.
// The refit state is derived at the first call and kept in r->refit; a failure to derive it leaves r->refit empty, and the next call
// tries again.  Returns cudaError_t as int.
int lbvh_refit(LbvhResult *r, const b200pt_vertex *d_verts, const uint32_t *d_indices, const DevMesh *d_meshes, const DevInstance *d_instances,
               uint32_t n_instances, cudaStream_t st);
// After the vertices of some meshes changed (d_verts holds them) and lbvh_refit ran: r->shade of every triangle of instances insts[0, m) is
// rewritten as lbvh_build writes it.  Both rebuilds recompute r->shade themselves.  d_list: device scratch of at least 2 m + 1 words.
// Returns cudaError_t as int.
int lbvh_refresh_shade(LbvhResult *r, const b200pt_vertex *d_verts, const uint32_t *d_indices, const DevMesh *d_meshes, const DevInstance *d_instances,
                       const DevInstance *h_instances, const DevMesh *h_meshes, const uint32_t *insts, uint32_t m, uint32_t *d_list, cudaStream_t st);
// *any = some float of d_v[0, n) is not finite.  d_flag: one device word of scratch; h_small: pinned host word for the readback.  Returns cudaError_t as int.
int any_nonfinite(const float *d_v, size_t n, uint32_t *d_flag, uint32_t *h_small, cudaStream_t st, bool *any);

// ---- glTF pose (pose_kernels.cu): skinned / morphed vertices from the rest data, written as b200pt_vertex records ----
// One descriptor per deformable mesh.  Its vertices are [vbase, vbase + count) of the rest data and of the output; its blocks of
// POSE_BLOCK threads start at block0.  Morph deltas are planes of count floats: for target t, plane (delta_base + (t * 8 + c) * count),
// c = 0..2 position, 3..5 normal, 6..7 uv.  Joints / weights: [vertex][4 * sets] from jw_base.
constexpr uint32_t POSE_BLOCK = 256;
constexpr uint32_t POSE_SMEM_JOINTS = 512;          // joint palettes up to this size are staged in shared memory (48 B per joint)
enum PoseFlags : uint32_t { POSE_SKINNED = 1, POSE_DPOS = 2, POSE_DNRM = 4, POSE_DUV = 8, POSE_GEN_NORMALS = 16 };
struct PoseMesh {
    uint32_t vbase, count, block0, flags;
    uint32_t sets, jw_base, n_joints, palette_base;   // palette_base: first joint of the mesh's palette (12 floats each)
    uint32_t targets, morph_base, ibase, _pad;        // morph_base: first weight; ibase: first index in the scene's index buffer
    size_t delta_base;
};
struct PoseDev {                                      // device arrays of the rest data, uploaded once per scene
    const PoseMesh *meshes; const uint32_t *block_mesh;
    const float *rest;                                // [vertex][8] position, NORMAL as stored, uv
    const uint32_t *joints; const float *weights; const float *deltas;
    const uint32_t *last_face;                        // per vertex (UINT32_MAX: none); generated-normal meshes only
    const uint32_t *indices;                          // the scene's index buffer
    const float *palette, *morph;                     // per pose
};
// out: vertex records at [vbase, ...), flag: set to 1 when a posed component is not finite (normals the loader leaves non-finite excepted).
// gen_normals: the second pass over the meshes loaded without NORMAL runs.  max_joints: the largest palette of a skinned mesh.  cudaError_t as int.
int launch_pose(const PoseDev &d, uint32_t n_blocks, uint32_t max_joints, bool gen_normals, b200pt_vertex *out, uint32_t *flag, cudaStream_t st);

// ---- post chain (post_kernels.cu) ----
struct PostParams { float Exposure, Gamma, BloomThreshold, BloomStrength, FalloffRange; };
void launch_accumulate(const float4 *frame, float4 *image, uint32_t first, uint32_t count, uint32_t frame_index, int grid, cudaStream_t st);   // running mean of pixels [first, first + count)
void launch_bloom_threshold(const float4 *hdr, float4 *mip0, uint32_t npix, PostParams p, int grid, cudaStream_t st);
// rows (optional): {first, end} row range of the destination the launch computes (multi-GPU post pass); nullptr = all rows
void launch_bloom_down(const float4 *src, uint32_t sw, uint32_t sh, float4 *dst, uint32_t dw, uint32_t dh, PostParams p, cudaStream_t st, const int *rows = nullptr);
// fused chain: threshold folded into the first down pass (mip 0 is never written) and [last up pass + threshold + tonemap] in one kernel
void launch_bloom_down_first(const float4 *hdr, uint32_t W, uint32_t H, float4 *mip1, uint32_t dw, uint32_t dh, PostParams p, cudaStream_t st, const int *rows = nullptr);
void launch_bloom_final(const float4 *hdr, const float4 *mip1, uint32_t mw, uint32_t mh, uchar4 *ldr, float4 *mip0_out, uint32_t W, uint32_t H, PostParams p, cudaStream_t st, const int *rows = nullptr);
void launch_bloom_up(const float4 *src, uint32_t sw, uint32_t sh, float4 *dst, uint32_t dw, uint32_t dh, PostParams p, cudaStream_t st, const int *rows = nullptr);
void launch_tonemap(const float4 *hdr, const float4 *bloom0, uchar4 *ldr, uint32_t W, uint32_t H, PostParams p, cudaStream_t st);
void launch_prepare_materials(DevMaterial *mats, uint32_t first, uint32_t count, cudaStream_t st);   // fills DevMaterial::pre0..pre3
// lut_baker.cu : kind 0 = reflect, 1 = refract hit-from-outside, 2 = refract hit-from-inside; partial holds slices * SX*SY*SZ floats
void launch_bake_lut(int kind, float *partial, float *table, uint32_t SX, uint32_t SY, uint32_t SZ, uint32_t sample_count, uint32_t seed,
                     uint32_t slices, cudaStream_t st);

} // namespace b200pt
