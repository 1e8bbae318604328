// engine.h -- host runtime: the CUDA counterparts of the reference's PathTracer (PathTracer/PathTracer.h:83-183)
// and PostProcessor (PathTracer/PostProcessor.h:25-33) classes.  One Engine == one GPU.
#pragma once
#include "host_api.h"
#include "kernels.h"
#include "cuda_resources.h"
#include <cuda_runtime.h>
#include <functional>

namespace b200pt {

class Engine {
public:
    explicit Engine(int device);
    ~Engine();

    // PathTracer::SetScene
    void set_scene(HostScene &&scene);
    void set_env_map(uint32_t w, uint32_t h, const float *rgba);
    void set_luts(const float *refl, const float *rout, const float *rin);

    void set_config(const b200pt_config &c);
    const b200pt_config &config() const { return cfg_; }
    void set_material(uint32_t idx, const b200pt_material &m);
    // TLAS::Update: count x 16 floats (b200pt_instance::Transform); rebuild: 0 refits in place, B200PT_REBUILD_GPU builds on the device (PLOC),
    // any other value builds the tree set_scene would build
    void update_instance_transforms(const float *transforms, uint32_t count, int rebuild);
    // the whole vertex array of each listed mesh (host or device memory), one refit / rebuild for the batch; rebuild as above
    void update_mesh_vertices(const b200pt_mesh_update *updates, uint32_t n, bool device, int rebuild);
    // glTF pose (DESIGN §15): the scene's nodes, skins and morph targets at time t of an animation (-1: the rest pose); the posed vertices of
    // the deformable meshes and every instance transform committed with one refit / rebuild (rebuild as above)
    void pose(int animation, float t, int rebuild);
    // PathTracer::AddVolume / SetVolume / RemoveVolume / SetPhaseFunction / AddDensityDataToVolume / RemoveDensityDataFromVolume (volumes.cuh)
    uint32_t add_volume(const b200pt_volume &v);
    void set_volume(uint32_t idx, const b200pt_volume &v);
    void remove_volume(uint32_t idx);
    void add_density_grid(uint32_t idx, const b200pt_density_grid &g);
    void remove_density_data(uint32_t idx);
    const std::vector<b200pt_volume> &volumes() const { return volumes_; }
    void set_phase_function(uint32_t pf);
    uint32_t phase_function() const { return phase_function_; }
    void set_atmosphere(const b200pt_atmosphere &a) { atmosphere_ = a; reset(); }     // parameters only (PathTracer.h:170-181); rendering with it is not built
    const b200pt_atmosphere &atmosphere() const { return atmosphere_; }
    const HostScene &scene() const { return scene_; }
    bool has_scene() const { return has_scene_; }
    bool has_env() const { return d_env_ && d_alias_ && d_env_row_cos_; }       // set_env_map has succeeded
    bool has_luts() const { return d_luts_[0] && d_luts_[1] && d_luts_[2]; }    // set_luts has succeeded
    // The device view of the scene that every launch reads, each field taken from the owner of its data or the host fact it depends on.
    // pre_pass is 0: path_trace sets it on its own copy.
    DevScene dev_scene() const;
    void set_camera(const float vi[16], const float pi[16]);
    void get_camera(float vi[16], float pi[16]) const;
    void resize(uint32_t w, uint32_t h);
    void reset();                                   // ResetPathTracing
    void set_partition(uint32_t rank, uint32_t world, uint32_t band);
    uint32_t width() const { return W_; }
    uint32_t height() const { return H_; }
    uint32_t local_rows() const { return local_rows_; }
    uint32_t samples_accumulated() const { return samples_accumulated_; }

    // adaptive sampling (no reference equivalent): per-pixel stop once the running mean has converged; any set resets the accumulation
    void set_adaptive(const b200pt_adaptive &a);
    const b200pt_adaptive &adaptive() const { return adaptive_; }
    void pixel_stats(uint32_t *counts, float *rel_error);   // local pixels: frames accumulated, relative standard error of the mean luminance
    uint32_t active_pixels();                               // local pixels still traced
    // per-pixel statistics without adaptive sampling: the same records, kept by k_resolve_adaptive over the identity list; any set resets the accumulation
    void set_track_variance(bool on);
    bool track_variance() const { return track_variance_; }

    // denoiser (no reference equivalent, denoise_kernels.cu): feature pass + a-trous filter into a buffer of its own; the accumulation is not touched
    void denoise(const b200pt_denoise_params &p, float *elapsed_ms);
    void get_denoised(float *dst, bool dst_is_device);
    void denoise_inputs(const b200pt_denoise_params &p, float *albedo_cov, float *normal_depth, float *variance);   // local rows, host memory
    void denoise_image(uint32_t w, uint32_t h, const float *color, const float *albedo_cov, const float *normal_depth, const float *variance,
                       const b200pt_denoise_params &p, float *out, bool is_device);
    void post_process_denoised();                           // the post chain on the denoised image

    // PathTracer::PathTrace x dispatches; returns true when all samples are accumulated (or, adaptive, no local pixel is active)
    bool path_trace(uint32_t dispatches, uint32_t base_seed);
    void synchronize();
    void flush() { check(cudaSetDevice(device_), "cudaSetDevice"); join_waves(); }   // device-side: the caller's stream waits for every launched wave
    void set_stream(cudaStream_t s);
    void set_profiling(bool on) { profiling_ = on; }
    void get_hdr(float *dst, bool dst_is_device);
    void set_hdr(const float *src, bool src_is_device);
    float4 *hdr_device() { return d_image_.get(); }
    // checkpoint / resume of the accumulation (SURVEY 5 "checkpoint / resume", 8f row 4): image + dispatch bookkeeping
    void save_checkpoint(const char *path);
    void load_checkpoint(const char *path);
    b200pt_counters counters();

    // PostProcessor
    void set_tonemap(const b200pt_tonemap &t) { tonemap_ = t; }
    void set_bloom(const b200pt_bloom &b) { bloom_ = b; }
    // HDR accumulate as a stand-alone pass (config 5): rows [y0, y1) of a full-size device frame are folded into the accumulation image (frame_index = frames already in it)
    void accumulate_rows(const float4 *d_frame, uint32_t frame_index, uint32_t y0, uint32_t y1);
    void post_input_rows(uint32_t y0, uint32_t y1, uint32_t *in0, uint32_t *in1);   // HDR rows that post_process_rows(y0, y1) reads
    void post_process();
    void post_process_rows(uint32_t y0, uint32_t y1);             // output rows [y0, y1) only (multi-GPU post pass); equals the same rows of post_process()
    void get_ldr_rows(uint32_t y0, uint32_t y1, uint8_t *dst, bool dst_is_device);   // device destination: asynchronous on the engine's stream
    void get_ldr(uint8_t *dst, bool dst_is_device);
    void get_bloom(float *dst);

    void volume_walks(uint32_t n, const float *org, const float *dir, const uint32_t *seeds, float ray_depth, float *T, float *scatter, int32_t *vol, uint32_t *rng2);
    void trace_closest(uint32_t n, const float *org, const float *dir, float tmin, float tmax, float *t, uint32_t *prim, uint32_t *inst, float *uv, uint32_t *stats = nullptr);
    // b200pt_trace_query (host arrays; see include/b200pt.h)
    void trace_query(int shape, int kind, bool fma, uint32_t n, const float *org, const float *dir, const float *tmin, const float *tmax, const uint32_t *target,
                     const float *tmax_test, float *t, uint32_t *prim, uint32_t *inst, float *uv, uint32_t *occluded, uint32_t *stats);
    // b200pt_shade_query (host arrays; see include/b200pt.h)
    void shade_query(bool force_general, uint32_t n, const uint32_t *inst, const uint32_t *prim, const float *uv, const float *dir, const float *org,
                     const float *pay_pdf, const uint32_t *rng, const float *L, float *out);
    // b200pt_miss_query (host arrays; see include/b200pt.h)
    void miss_query(uint32_t n, const float *dir, const uint32_t *depth, const float *pay_pdf, float *out);
    // b200pt_bounce_query (host arrays; see include/b200pt.h): one bounce of path_trace's loop for caller-given paths
    void bounce_query(uint32_t n, const float *in, uint32_t flags, float *out, uint32_t *survivors);
    void scene_stats(uint32_t *tris, uint32_t *nodes, uint32_t *emissive, uint32_t *textures) const;
    // b200pt_bvh2_ploc_build_query (host arrays; see include/b200pt.h): the device builder and the device collapse on the caller's boxes
    void ploc_build_query(const float *ref_boxes, uint32_t n, BvhNode *nodes_out, uint32_t *perm_out, uint32_t *n_out, int *depth_out,
                          Bvh4Node *nodes4_out, uint32_t *n4_out, int *depth4_out);
    void bake_lut(int kind, uint32_t sx, uint32_t sy, uint32_t sz, uint32_t sample_count, uint32_t seed, uint32_t slices, float *out_host, float *elapsed_ms);

    std::string last_error;

private:
    // The acceleration structure and what is decided when it is built: the launch configuration and the flat walk (B200PT_FLAT_MAX).
    struct SceneTree {
        LbvhResult bvh{}; LaunchCfg lc{}; uint32_t n_flat = 0;
        void view(DevScene &sc) const;              // the tree's fields of a DevScene
    };
    void free_scene();
    void upload_scene();
    void fill_instances();                          // h_instances_ and n_tris_ from scene_.instances
    void upload_instances();                        // d_instances_ from h_instances_ (o2w / w2o, emissive_tri_count)
    SceneTree build_bvh(bool gpu_builder = false);  // the BVH half of upload_scene
    void rebuild_emissive();
    void rebuild_tri_class();                       // per-triangle shading class (MaterialClass) + the set of classes present in the scene
    void upload_volumes();
    DevMaterial make_dev_material(const b200pt_material &m) const;
    void ensure_image();
    void ensure_wave(size_t capacity, int contexts);
    void free_wave();
    void ensure_post();
    void free_post();
    DevConfig make_dev_config() const;
    void check(cudaError_t e, const char *what) const;

    int device_;
    Stream own_stream_, aux_stream_[2];             // declared first: destroyed after every member that may still be in use on them
    cudaStream_t stream_ = nullptr;                 // own_stream_ or the caller's (set_stream)
    bool profiling_ = false;
    std::vector<Event> prof_ev_;
    Event ev_[2];
    bool timed_ = false;                            // ev_ have been recorded (by a path_trace call that launched work)

    HostScene scene_;
    bool has_scene_ = false;
    b200pt_config cfg_;
    float view_inv_[16], proj_inv_[16];
    uint32_t W_ = 0, H_ = 0, rank_ = 0, world_ = 1, band_ = 16, local_rows_ = 0;
    uint64_t dispatch_count_ = 0;
    uint32_t frame_count_ = 0, samples_accumulated_ = 0;

    // device scene (dev_scene() is its view)
    DevPtr<b200pt_vertex> d_verts_; DevPtr<uint32_t> d_indices_; DevPtr<DevMesh> d_meshes_; DevPtr<DevInstance> d_instances_;
    DevPtr<DevMaterial> d_materials_; DevPtr<DevTexture> d_textures_; DevPtr<DevEmissive> d_emissive_; DevPtr<EmTri> d_em_tris_; DevPtr<uint32_t> d_em_tri_base_;
    std::vector<DevPtr<uint8_t>> d_texdata_;
    std::vector<DevInstance> h_instances_; std::vector<DevMesh> h_meshes_;
    DevPtr<float4> d_env_; DevPtr<uint2> d_alias_; DevPtr<float2> d_env_row_cos_; uint32_t env_w_ = 0, env_h_ = 0; DevPtr<float> d_luts_[3];
    std::vector<b200pt_volume> volumes_; uint32_t phase_function_ = 0; DevPtr<DevVolume> d_volumes_;
    struct GridData { PreparedGrid host; DevPtr<float> d_values, d_max_densities; };
    std::vector<std::shared_ptr<GridData>> grids_;      // parallel to volumes_: density data of the heterogeneous ones (nullptr: homogeneous)
    DevPtr<DevGrid> d_grids_; int density_data_counter_ = 0;   // PathTracer.cpp:1508-1513: slots are handed out round-robin
    b200pt_atmosphere atmosphere_{};
    SceneTree tree_{};
    PinnedPtr<uint32_t> h_small_;                   // pinned 4-word readback buffer of the GPU tree builder (ploc.cu)
    DevPtr<uint8_t> d_scratch_; size_t scratch_bytes_ = 0;   // scratch(): the staging buffer and shading-refresh list of update_mesh_vertices and pose
    void *scratch(size_t bytes);
    // the commit of update_instance_transforms, update_mesh_vertices and pose: the listed meshes' whole vertex arrays (host memory, or device
    // memory on the stream) and, when given, every instance transform; one refit / rebuild; ResetPathTracing.  A failure restores both.
    struct VertexSource { uint32_t mesh; const b200pt_vertex *data; bool device; };
    void commit(const std::vector<VertexSource> &src, const std::vector<b200pt_instance> *instances, int rebuild);
    // rest data of the deformable meshes of a glTF scene (pose_kernels.cu), uploaded by set_scene; nothing for other scenes
    void upload_pose_data();
    void free_pose_data();
    DeviceBlocks pose_blocks_;                      // every device allocation behind pose_dev_
    PoseDev pose_dev_{};
    std::vector<PoseMesh> pose_meshes_;             // HostAnimation::deformable order
    uint32_t pose_grid_ = 0, pose_max_joints_ = 0, pose_vertices_ = 0, pose_palette_floats_ = 0, pose_morph_floats_ = 0;
    bool pose_gen_normals_ = false;
    uint32_t n_tris_ = 0, n_emissive_ = 0;
    DevPtr<uint8_t> d_tri_class_; uint32_t class_mask_ = 0;   // bit c: some triangle's material is of MaterialClass c

    // framebuffer + post
    DevPtr<float4> d_image_; size_t image_pixels_ = 0;
    b200pt_tonemap tonemap_{ 1.0f, 2.2f };
    b200pt_bloom bloom_{ 2.0f, 1.0f, 10, 5.0f };
    std::vector<DevPtr<float4>> d_mips_; std::vector<uint32_t> mip_wh_; DevPtr<uchar4> d_ldr_; uint32_t post_w_ = 0, post_h_ = 0;
    bool keep_bloom_ = false, bloom_valid_ = false;   // fused post chain: mip 0 is written only once get_bloom() has been used

    // wave buffers: one context per wave in flight.  Two contexts on two internal streams let the latency-bound tail of wave w (late bounces: few, long rays)
    // overlap the full-machine head of wave w+1; k_resolve runs in dispatch order (events), so the image does not depend on it.
    struct WaveBuf {
        DeviceBlocks arrays;                        // the cap-sized arrays below, from ps to q_miss
        PathState ps[2]{}; ShadeOut so{};
        float4 *sample_buf = nullptr; uint32_t *rng_carry = nullptr; uint32_t *q_hit = nullptr, *q_miss = nullptr;
        DevPtr<uint32_t> counts; PinnedPtr<uint32_t> h_count;
        DevPtr<DevDispatch> d_disp; PinnedPtr<DevDispatch> h_disp; Event disp_ev;   // this context's slice of the dispatch table (pinned host copy reusable once disp_ev has fired)
        size_t cap = 0;
    };
    WaveBuf wb_[2];
    Event resolved_ev_[2], image_free_ev_;
    uint64_t wave_seq_ = 0;                         // waves launched so far: wave w runs in context w & 1 and resolves after wave w - 1
    size_t wave_cap_ = 0;                           // capacity (paths) of every allocated context
    void sync_all();                                // the caller's stream AND the internal wave streams are idle
    void join_waves();                              // work enqueued on the caller's stream from here on sees every launched wave resolved into the image
    DevPtr<WaveCounters> d_ctr_;
    b200pt_counters last_{};
    bool scene_has_media() const;                   // can a path random-walk inside a mesh without gaining Depth?
    // bounce k of a sub-wave in context B: the paths of pst[cur] (control word k & 1) are traced and shaded, the survivors written to
    // pst[cur ^ 1].  mark(kind) follows each launch group (profiling).  Returns the number of kernels enqueued on st.
    uint64_t bounce(const CallPlan &cp, const DevScene &sc, const DevConfig &dc, WaveBuf &B, const PathState pst[2], int cur, uint32_t k, uint32_t flags, cudaStream_t st,
                    const std::function<void(int)> &mark);

    // adaptive sampling: allocated only while enabled.  The state is rebuilt lazily (prepare_adaptive) after every reset.
    b200pt_adaptive adaptive_{};
    DevPtr<uint4> d_px_state_;                      // one record per local pixel (kernels.h: meanL, M2, n_p, flags)
    DevPtr<uint32_t> d_active_, d_tile_count_, d_active_count_; PinnedPtr<uint32_t> h_active_count_;
    size_t adaptive_pixels_ = 0;                    // local pixels the buffers were sized for
    uint32_t active_count_ = 0;                     // A: entries of d_active_ (host copy, read back at every interval boundary)
    bool adaptive_ready_ = false;                   // the state matches the accumulation (false after reset)
    void prepare_adaptive();
    void free_adaptive();
    void update_active(bool decide, cudaStream_t st);   // decision / list rebuild on st, then A read back (blocks the host)
    bool track_variance_ = false;                   // the records without adaptive sampling (set_track_variance)
    bool records() const { return adaptive_.Enable != 0u || track_variance_; }

    // denoiser: one allocation of W * local_rows pixels = [features 2n float4 | denoised n float4 | filter scratch 3n float4 | variance n float]
    DevPtr<float4> d_dn_; size_t dn_pixels_ = 0;
    uint32_t dn_w_ = 0, dn_h_ = 0;                  // size of the image the denoised buffer holds (0: none)
    DevPtr<float4> d_dn_img_; size_t dn_img_bytes_ = 0;   // denoise_image: filter scratch (+ device copies of host arrays)
    bool post_denoised_ = false;                    // the last post pass read the denoised image (get_bloom re-runs it on the same input)
    void ensure_denoise();
    void free_denoise();
    bool has_denoised() const { return d_dn_ && dn_w_ == W_ && dn_h_ == H_; }
    void run_features(const b200pt_denoise_params &p);   // features + variance of the local rows into d_dn_
    void post_chain(const float4 *src, uint32_t y0, uint32_t y1);
};

} // namespace b200pt
