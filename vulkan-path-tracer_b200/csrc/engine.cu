// engine.cu -- host runtime of the wavefront path tracer (see engine.h).
// Orchestration per b200pt_path_trace call (all on one CUDA stream, no host sync inside a wave unless the
// scene can scatter inside a medium or MaxDepth is large enough that early exit pays):
//   upload dispatch table -> for each wave of F dispatches: raygen -> [extend, shade, connect] x bounces -> resolve
// (adaptive sampling: the waves of each interval trace the active pixels only; k_adaptive_update + one 4-byte read-back at its end)
#include "engine.h"
#include <cstring>
#include <cstdio>
#include <algorithm>
#include <cmath>

namespace b200pt {

static void check_cuda(cudaError_t e, const char *what) {
    if (e != cudaSuccess) throw CudaError{ (int)e, std::string(what) + ": " + cudaGetErrorString(e) };
}
void Engine::check(cudaError_t e, const char *what) const { check_cuda(e, what); }
#define CK(x) check((x), #x)

static const uint32_t kMaxDispatchTable = 1u << 16;

static Event make_event(unsigned flags) {
    cudaEvent_t e = nullptr;
    check_cuda(cudaEventCreateWithFlags(&e, flags), "cudaEventCreateWithFlags");
    return Event(e);
}
static Stream make_stream() {
    cudaStream_t s = nullptr;
    check_cuda(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), "cudaStreamCreateWithFlags");
    return Stream(s);
}

Engine::Engine(int device) : device_(device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) throw CudaError{ B200PT_ERR_NO_DEVICE, "no CUDA device available (the product has no CPU fallback)" };
    if (device < 0 || device >= n) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "device ordinal out of range" };
    CK(cudaSetDevice(device_));
    own_stream_ = make_stream(); stream_ = own_stream_.get();
    ev_[0] = make_event(cudaEventDefault); ev_[1] = make_event(cudaEventDefault);
    b200pt_default_config(&cfg_);
    memset(view_inv_, 0, sizeof view_inv_); memset(proj_inv_, 0, sizeof proj_inv_);
    for (int i = 0; i < 4; i++) view_inv_[i * 5] = proj_inv_[i * 5] = 1.0f;
    CK(alloc(d_ctr_, sizeof(WaveCounters)));
    CK(cudaMemset(d_ctr_.get(), 0, sizeof(WaveCounters)));
    for (int c = 0; c < 2; c++) {
        CK(alloc(wb_[c].counts, CTRL_WORDS * sizeof(uint32_t))); CK(alloc(wb_[c].h_count, 4 * sizeof(uint32_t)));
        aux_stream_[c] = make_stream(); resolved_ev_[c] = make_event(cudaEventDisableTiming);
        wb_[c].disp_ev = make_event(cudaEventDisableTiming);
        CK(alloc(wb_[c].d_disp, kMaxDispatchTable * sizeof(DevDispatch))); CK(alloc(wb_[c].h_disp, kMaxDispatchTable * sizeof(DevDispatch)));
    }
    image_free_ev_ = make_event(cudaEventDisableTiming);
    CK(alloc(h_active_count_, sizeof(uint32_t)));
    CK(alloc(h_small_, 4 * sizeof(uint32_t)));
    b200pt_default_adaptive(&adaptive_);
    b200pt_default_atmosphere(&atmosphere_);
    memset(&last_, 0, sizeof last_);
}

// The members release everything else after this body, the streams last.
Engine::~Engine() {
    cudaSetDevice(device_);
    for (auto &st : aux_stream_) if (st) cudaStreamSynchronize(st.get());
    if (stream_) cudaStreamSynchronize(stream_);
}

// Device scratch of the engine, grown on demand and kept: the per-frame updates allocate (and free, which synchronises the device) nothing.
// Only valid until the next call; the caller has synchronised the work that used the previous contents.
void *Engine::scratch(size_t bytes) {
    if (bytes > scratch_bytes_) {
        scratch_bytes_ = 0;
        CK(alloc(d_scratch_, bytes)); scratch_bytes_ = bytes;
    }
    return d_scratch_.get();
}

void Engine::sync_all() {
    for (auto &st : aux_stream_) if (st) CK(cudaStreamSynchronize(st.get()));
    CK(cudaStreamSynchronize(stream_));
}
void Engine::join_waves() {
    if (wave_seq_ == 0) return;
    for (auto &e : resolved_ev_) CK(cudaStreamWaitEvent(stream_, e.get(), 0));    // an event that was never recorded counts as complete
}

void Engine::free_scene() {
    d_verts_.reset(); d_indices_.reset(); d_meshes_.reset(); d_instances_.reset(); d_materials_.reset(); d_textures_.reset(); d_emissive_.reset();
    d_em_tris_.reset(); d_em_tri_base_.reset(); d_tri_class_.reset();
    d_texdata_.clear();
    tree_ = {};
    free_pose_data();
    has_scene_ = false;
}

// PathTracer::SetScene (PathTracer.cpp:158-676)
void Engine::set_scene(HostScene &&scene) {
    CK(cudaSetDevice(device_));
    sync_all();
    free_scene();
    scene_ = std::move(scene);
    // capacity limits of the reference (PathTracer.h:192-195, asserts PathTracer.cpp:182-184)
    if (scene_.meshes.size() >= 10000 || scene_.materials.size() >= 10000 || scene_.instances.size() >= 100000)
        throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "scene exceeds the reference's MAX_ENTITIES / MAX_INSTANCES limits" };
    upload_scene();
    // camera: PathTracer.cpp:187-188,578 then the Editor/FlyCamera round trip
    camera_from_view(scene_.camera_view, scene_.camera_aspect, view_inv_, proj_inv_);
    // output image: W = (uint)(1080 * aspect), H = 1080 (PathTracer.cpp:509-512)
    W_ = (uint32_t)((float)1080 * scene_.camera_aspect); H_ = 1080;
    local_rows_ = partition_local_rows(H_, rank_, world_, band_);
    ensure_image();
    has_scene_ = true;
    reset();
}

void Engine::upload_scene() {
    size_t nv = 0, ni = 0;
    h_meshes_.clear();
    for (auto &m : scene_.meshes) { h_meshes_.push_back({ (uint32_t)nv, (uint32_t)ni, (uint32_t)(m.indices.size() / 3), 0 }); nv += m.vertices.size(); ni += m.indices.size(); }
    std::vector<b200pt_vertex> verts(nv); std::vector<uint32_t> idx(ni);
    for (size_t i = 0; i < scene_.meshes.size(); i++) {
        memcpy(&verts[h_meshes_[i].vbase], scene_.meshes[i].vertices.data(), scene_.meshes[i].vertices.size() * sizeof(b200pt_vertex));
        memcpy(&idx[h_meshes_[i].ibase], scene_.meshes[i].indices.data(), scene_.meshes[i].indices.size() * 4);
    }
    CK(alloc(d_verts_, nv * sizeof(b200pt_vertex))); CK(cudaMemcpy(d_verts_.get(), verts.data(), nv * sizeof(b200pt_vertex), cudaMemcpyHostToDevice));
    CK(alloc(d_indices_, ni * 4)); CK(cudaMemcpy(d_indices_.get(), idx.data(), ni * 4, cudaMemcpyHostToDevice));
    CK(alloc(d_meshes_, h_meshes_.size() * sizeof(DevMesh))); CK(cudaMemcpy(d_meshes_.get(), h_meshes_.data(), h_meshes_.size() * sizeof(DevMesh), cudaMemcpyHostToDevice));
    fill_instances();
    CK(alloc(d_instances_, h_instances_.size() * sizeof(DevInstance)));
    {
        std::vector<DevMaterial> dm; dm.reserve(scene_.materials.size());
        for (const auto &m : scene_.materials) dm.push_back(make_dev_material(m));
        CK(alloc(d_materials_, dm.size() * sizeof(DevMaterial)));
        CK(cudaMemcpy(d_materials_.get(), dm.data(), dm.size() * sizeof(DevMaterial), cudaMemcpyHostToDevice));
        launch_prepare_materials(d_materials_.get(), 0, (uint32_t)dm.size(), stream_);
        CK(cudaStreamSynchronize(stream_));
    }
    CK(alloc(d_emissive_, std::max<size_t>(1, scene_.instances.size()) * sizeof(DevEmissive)));
    rebuild_emissive();
    upload_instances();
    // textures
    std::vector<DevTexture> dt(scene_.textures.size());
    d_texdata_.resize(scene_.textures.size());
    for (size_t i = 0; i < scene_.textures.size(); i++) {
        const HostTexture &t = scene_.textures[i];
        CK(alloc(d_texdata_[i], std::max<size_t>(t.data.size(), 4)));
        CK(cudaMemcpy(d_texdata_[i].get(), t.data.data(), t.data.size(), cudaMemcpyHostToDevice));
        dt[i] = { d_texdata_[i].get(), t.width, t.height, t.channels, 0 };
    }
    CK(alloc(d_textures_, dt.size() * sizeof(DevTexture))); CK(cudaMemcpy(d_textures_.get(), dt.data(), dt.size() * sizeof(DevTexture), cudaMemcpyHostToDevice));
    CK(alloc(d_tri_class_, std::max<size_t>(1, n_tris_)));
    rebuild_tri_class();
    tree_ = build_bvh();
    upload_pose_data();
}

void Engine::upload_instances() {
    CK(cudaMemcpy(d_instances_.get(), h_instances_.data(), h_instances_.size() * sizeof(DevInstance), cudaMemcpyHostToDevice));
}

// DevInstance of every instance from scene_.instances (o2w = rows 0-2 of the column-major Transform, w2o its inverse); emissive_tri_count is
// rebuild_emissive's.  set_scene and update_instance_transforms both use it.
void Engine::fill_instances() {
    // instances: one per MeshInstance in loader order == InstanceIndex (TLASImpl.cpp:29-35)
    h_instances_.assign(scene_.instances.size(), DevInstance{});
    uint32_t tri_base = 0;
    for (size_t i = 0; i < scene_.instances.size(); i++) {
        const b200pt_instance &in = scene_.instances[i]; DevInstance &d = h_instances_[i];
        for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) d.o2w[r * 4 + c] = in.Transform[c * 4 + r];
        mat3_inverse_from_o2w(d.o2w, d.w2o);
        d.mesh = in.MeshIndex; d.material = in.MaterialIndex; d.tri_base = tri_base;
        tri_base += h_meshes_[in.MeshIndex].tri_count;
    }
    n_tris_ = tri_base;
}

// The acceleration structure of the instances in d_instances_ and its launch configuration.  set_scene and update_instance_transforms(rebuild)
// both use it.  gpu_builder: the tree is built on the device (PLOC over the LBVH's references, ploc.cu) instead of by the host tree-quality passes.
Engine::SceneTree Engine::build_bvh(bool gpu_builder) {
    SceneTree tree;
    LbvhResult *const out = &tree.bvh;
    // acceleration structure: GPU LBVH over the flattened instances
    // tree-quality pass over the GPU LBVH: same hits, fewer node visits / triangle tests.  Level 3 (full binned-SAH build + insertion-based
    // refinement) is the default;
    // B200PT_BVH_SAH=0..5 overrides (0 = plain LBVH).
    int sah_mode = 3;
    if (const char *e = getenv("B200PT_BVH_SAH")) sah_mode = (e[0] >= '0' && e[0] <= '5' && e[1] == 0) ? e[0] - '0' : 3;
    if (gpu_builder) sah_mode = 0;
    std::vector<float> host_ref_box; DevPtr<float> ref_box;                 // inputs of the tree passes below, released when the build ends
    int r = lbvh_build(d_verts_.get(), d_indices_.get(), d_meshes_.get(), d_instances_.get(), (uint32_t)h_instances_.size(), n_tris_, out, stream_,
                       sah_mode == 2 || sah_mode == 3 ? &host_ref_box : nullptr, gpu_builder ? &ref_box : nullptr);
    if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("lbvh_build failed: ") + cudaGetErrorString((cudaError_t)r) };
    if (gpu_builder) {
        r = lbvh_ploc_rebuild(out, std::move(ref_box), h_small_.get(), stream_);
        if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("lbvh_ploc_rebuild failed: ") + cudaGetErrorString((cudaError_t)r) };
    }
    if (sah_mode) {
        double sah[2];
        r = lbvh_refine_sah(out, host_ref_box.empty() ? nullptr : host_ref_box.data(), stream_, sah, sah_mode);
        if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("lbvh_refine_sah failed: ") + cudaGetErrorString((cudaError_t)r) };
        if (getenv("B200PT_DEBUG")) fprintf(stderr, "[b200pt] SAH pass (mode %d): cost %.3f -> %.3f, depth %d\n", sah_mode, sah[0], sah[1], out->max_depth);
    }
    if (out->bytes > 64u * 1024u) {                                         // scenes that traverse out of L2/HBM get the BVH4 (host collapse of the GPU-built BVH2)
        r = gpu_builder ? lbvh_build_wide_device(out, h_small_.get(), stream_) : lbvh_build_wide(out, stream_);
        if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("lbvh_build_wide failed: ") + cudaGetErrorString((cudaError_t)r) };
    }
    // A handful of triangle slots (the 12-triangle Cornell box): shared-memory traversals test them in order, no hierarchy (bvh_traverse.cuh).
    {
        uint32_t flat_max = 16;
        if (const char *e = getenv("B200PT_FLAT_MAX")) { const int v = atoi(e); if (v >= 0 && v <= 64) flat_max = (uint32_t)v; }
        tree.n_flat = (out->n_tris <= flat_max) ? out->n_tris : 0u;
    }
    DevScene sc{};
    tree.view(sc);
    int q = query_launch_cfg(sc, out->max_depth, out->depth4, &tree.lc);
    if (q != 0) throw CudaError{ B200PT_ERR_CUDA, "query_launch_cfg failed" };
    return tree;
}

void Engine::SceneTree::view(DevScene &sc) const {
    sc.nodes = bvh.nodes.get(); sc.tris = bvh.tris; sc.shade_tris = bvh.shade.get(); sc.tri_slot = bvh.tri_slot.get();
    sc.n_tris = bvh.n_tris; sc.n_nodes = bvh.n_nodes; sc.root = bvh.root; sc.bvh_bytes = bvh.bytes <= 0xFFFFFFFFull ? (uint32_t)bvh.bytes : 0;
    sc.nodes4 = bvh.nodes4.get(); sc.n_nodes4 = bvh.n_nodes4;
    sc.n_flat = n_flat;
}

// TLAS::Update (VulkanHelper/Source/Vulkan/TLASImpl.cpp:192-293): every instance transform replaced, the tree refit in place (rebuild == 0),
// built anew on the device (B200PT_REBUILD_GPU) or as set_scene would build it (any other value); then ResetPathTracing.  Camera, config, image size, partition, materials, volumes and the
// environment stay.  Every argument is checked before anything changes.  A failed update restores the previous transforms: a failed rebuild keeps
// the previous tree, a failed refit refits the tree back to them (and if that fails too, the handle has no scene until the next set_scene).
void Engine::update_instance_transforms(const float *xf, uint32_t count, int rebuild) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!xf || count != scene_.instances.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "transform count differs from the instance count" };
    for (size_t i = 0; i < (size_t)count * 16; i++) if (!std::isfinite(xf[i])) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "transform entry is not finite" };
    sync_all();                                                 // the waves in flight neither read a half-updated tree nor resolve into the new accumulation
    std::vector<b200pt_instance> moved = scene_.instances;
    for (uint32_t i = 0; i < count; i++) memcpy(moved[i].Transform, xf + (size_t)i * 16, sizeof moved[i].Transform);
    commit({}, &moved, rebuild);
}

// Mesh vertex update (no reference equivalent): the whole vertex array of each listed mesh replaced in d_verts_ and in the host mirror
// scene_.meshes (rebuild_emissive, set_material, the instance update and get_mesh_vertices read it), the emissive records rebuilt from the
// mirror, then the tree refit in place with the shading records of the changed meshes' instances rewritten (rebuild == 0), or built anew as
// update_instance_transforms builds it; then ResetPathTracing.  What stays and how a failure is undone: as update_instance_transforms.
// Every argument is checked before anything changes; device input is staged in one buffer and checked there first.
void Engine::update_mesh_vertices(const b200pt_mesh_update *u, uint32_t n, bool device, int rebuild) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!u || n == 0) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "no mesh update" };
    std::vector<uint8_t> listed(scene_.meshes.size(), 0);
    size_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (u[i].mesh >= scene_.meshes.size() || listed[u[i].mesh]) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "mesh index out of range or repeated" };
        listed[u[i].mesh] = 1;
        if (!u[i].vertices) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "null vertex pointer" };
        if (u[i].vertex_count != scene_.meshes[u[i].mesh].vertices.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "vertex count differs from the mesh's" };
        total += u[i].vertex_count;
    }
    constexpr size_t VB = sizeof(b200pt_vertex), VF = VB / sizeof(float);
    if (!device)
        for (uint32_t i = 0; i < n; i++) {
            const float *f = reinterpret_cast<const float *>(u[i].vertices);
            for (size_t k = 0; k < (size_t)u[i].vertex_count * VF; k++) if (!std::isfinite(f[k])) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "vertex component is not finite" };
        }
    sync_all();                                                 // the waves in flight neither read half-updated records nor resolve into the new accumulation
    std::vector<VertexSource> src(n);
    b200pt_vertex *stage = nullptr;                             // device input: [update 0 | update 1 | ... | flag word]
    if (device) {
        stage = static_cast<b200pt_vertex *>(scratch(total * VB + 16));
        size_t o = 0;
        for (uint32_t i = 0; i < n; o += u[i].vertex_count, i++)
            if (u[i].vertex_count) CK(cudaMemcpyAsync(stage + o, u[i].vertices, u[i].vertex_count * VB, cudaMemcpyDeviceToDevice, stream_));
        bool bad = false;
        const int r = any_nonfinite(reinterpret_cast<const float *>(stage), total * VF, reinterpret_cast<uint32_t *>(stage + total), h_small_.get(), stream_, &bad);
        if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("any_nonfinite failed: ") + cudaGetErrorString((cudaError_t)r) };
        if (bad) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "vertex component is not finite" };
    }
    size_t o = 0;
    for (uint32_t i = 0; i < n; o += u[i].vertex_count, i++) src[i] = { u[i].mesh, device ? stage + o : u[i].vertices, device };
    commit(src, nullptr, rebuild);
}

// The listed vertex arrays replaced in d_verts_ and the host mirror scene_.meshes, and (instances != nullptr) every instance transform replaced
// (d_instances_ / h_instances_ through fill_instances); the emissive records rebuilt from the mirror; then the tree refit in place, with the
// shading records of the changed meshes' instances rewritten (rebuild == 0), built on the device (B200PT_REBUILD_GPU) or as set_scene would
// build it (any other value); then ResetPathTracing.  The caller has checked everything and synchronised the waves in flight.  A failure
// restores the previous vertices and transforms: a failed rebuild keeps the previous tree, a failed refit refits the tree back to them (and if
// that fails too, the handle has no scene until the next set_scene).
void Engine::commit(const std::vector<VertexSource> &src, const std::vector<b200pt_instance> *instances, int rebuild) {
    constexpr size_t VB = sizeof(b200pt_vertex);
    std::vector<uint8_t> listed(scene_.meshes.size(), 0);
    for (const VertexSource &s : src) listed[s.mesh] = 1;
    std::vector<std::vector<b200pt_vertex>> old(src.size());
    for (size_t i = 0; i < src.size(); i++) old[i] = scene_.meshes[src[i].mesh].vertices;
    const std::vector<b200pt_instance> old_instances = instances ? scene_.instances : std::vector<b200pt_instance>();
    auto restore = [&]() {
        for (size_t i = 0; i < src.size(); i++) {
            std::vector<b200pt_vertex> &mv = scene_.meshes[src[i].mesh].vertices;
            mv = old[i];
            if (!mv.empty()) CK(cudaMemcpyAsync(d_verts_.get() + h_meshes_[src[i].mesh].vbase, mv.data(), mv.size() * VB, cudaMemcpyHostToDevice, stream_));
        }
        if (instances) { scene_.instances = old_instances; fill_instances(); }
        CK(cudaStreamSynchronize(stream_));
        rebuild_emissive();                                     // DevEmissive::xf, the world-space EmTri
        upload_instances();
    };
    try {
        for (const VertexSource &s : src) {
            std::vector<b200pt_vertex> &mv = scene_.meshes[s.mesh].vertices;
            b200pt_vertex *dst = d_verts_.get() + h_meshes_[s.mesh].vbase;
            const size_t bytes = mv.size() * VB;
            if (!bytes) continue;
            if (s.device) {
                CK(cudaMemcpyAsync(dst, s.data, bytes, cudaMemcpyDeviceToDevice, stream_));
                CK(cudaMemcpyAsync(mv.data(), s.data, bytes, cudaMemcpyDeviceToHost, stream_));   // the mirror: the updated ranges only
            } else {
                memcpy(mv.data(), s.data, bytes);
                CK(cudaMemcpyAsync(dst, mv.data(), bytes, cudaMemcpyHostToDevice, stream_));
            }
        }
        if (instances) { scene_.instances = *instances; fill_instances(); }
        CK(cudaStreamSynchronize(stream_));
        rebuild_emissive();                                     // the world-space EmTri, from the mirror
        upload_instances();
    } catch (...) {
        try { restore(); } catch (...) { has_scene_ = false; }
        throw;
    }
    if (!rebuild) {
        std::vector<uint32_t> changed;                          // instances of the updated meshes: their shading records are rewritten
        for (size_t a = 0; a < h_instances_.size(); a++) if (listed[h_instances_[a].mesh]) changed.push_back((uint32_t)a);
        uint32_t *const d_list = src.empty() ? nullptr : static_cast<uint32_t *>(scratch((2 * changed.size() + 1) * sizeof(uint32_t)));
        auto refit = [&]() {
            int r = lbvh_refit(&tree_.bvh, d_verts_.get(), d_indices_.get(), d_meshes_.get(), d_instances_.get(), (uint32_t)h_instances_.size(), stream_);
            if (r == 0 && !src.empty())
                r = lbvh_refresh_shade(&tree_.bvh, d_verts_.get(), d_indices_.get(), d_meshes_.get(), d_instances_.get(), h_instances_.data(), h_meshes_.data(), changed.data(),
                                       (uint32_t)changed.size(), d_list, stream_);
            return r;
        };
        const int r = refit();
        if (r != 0) {                                           // back to the previous state, and the tree refit to it
            try { restore(); if (refit() != 0) has_scene_ = false; } catch (...) { has_scene_ = false; }
            throw CudaError{ B200PT_ERR_CUDA, std::string("lbvh_refit failed: ") + cudaGetErrorString((cudaError_t)r) };
        }
    } else {
        SceneTree fresh;
        try { fresh = build_bvh(rebuild == B200PT_REBUILD_GPU); }
        catch (...) { try { restore(); } catch (...) { has_scene_ = false; } throw; }
        tree_ = std::move(fresh);
    }
    reset();
}

// The rest data of the deformable meshes (HostAnimation::deformable), in device memory until the next set_scene: rest vertices, joints and
// weights of every set, morph deltas as planes (PoseMesh), the last face of each vertex of generated-normal meshes, and room for one pose's
// joint palettes and morph weights.  Scenes without deformable meshes allocate nothing.
void Engine::upload_pose_data() {
    pose_meshes_.clear(); pose_grid_ = pose_max_joints_ = pose_vertices_ = pose_palette_floats_ = pose_morph_floats_ = 0; pose_gen_normals_ = false;
    if (!scene_.animation || scene_.animation->deformable.empty()) return;
    const HostAnimation &A = *scene_.animation;
    size_t nv = 0, njw = 0, ndelta = 0;
    std::vector<uint32_t> block_mesh;
    for (int p : A.deformable) {
        const AnimPrim &ap = A.prims[p];
        PoseMesh m{};
        const int skin = A.prim_skin[p];
        const bool ok = ap.err.empty() && !ap.rest.empty();    // a mesh with bad data is never posed (evaluate_pose rejects it): no rest data
        m.vbase = (uint32_t)nv; m.count = ok ? ap.count : 0; m.block0 = (uint32_t)block_mesh.size();
        m.flags = (skin >= 0 ? POSE_SKINNED : 0) | (!ap.dpos.empty() ? POSE_DPOS : 0) | (!ap.dnrm.empty() ? POSE_DNRM : 0) | (!ap.duv.empty() ? POSE_DUV : 0) |
                  (ap.gen_normals ? POSE_GEN_NORMALS : 0);
        m.sets = skin >= 0 ? ap.sets : 0; m.jw_base = (uint32_t)njw;
        m.n_joints = skin >= 0 ? (uint32_t)A.skins[skin].joints.size() : 0; m.palette_base = pose_palette_floats_ / 12;
        m.targets = ap.targets; m.morph_base = pose_morph_floats_; m.ibase = h_meshes_[p].ibase; m.delta_base = ndelta;
        pose_meshes_.push_back(m);
        for (uint32_t b = 0; b < (m.count + POSE_BLOCK - 1) / POSE_BLOCK; b++) block_mesh.push_back((uint32_t)pose_meshes_.size() - 1);
        nv += m.count; njw += (size_t)m.count * 4 * m.sets; ndelta += (size_t)m.count * 8 * (m.flags & (POSE_DPOS | POSE_DNRM | POSE_DUV) ? m.targets : 0);
        pose_palette_floats_ += m.n_joints * 12; pose_morph_floats_ += m.targets;
        pose_max_joints_ = std::max(pose_max_joints_, m.n_joints);
        if (m.flags & POSE_GEN_NORMALS) pose_gen_normals_ = true;
    }
    if (nv > 0xFFFFFFFFull / 8) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "too many deformable vertices" };
    std::vector<float> rest(nv * 8), weights(njw), deltas(ndelta, 0.0f);
    std::vector<uint32_t> joints(njw), last_face(nv, UINT32_MAX);
    for (size_t d = 0; d < pose_meshes_.size(); d++) {
        const PoseMesh &m = pose_meshes_[d]; const AnimPrim &ap = A.prims[A.deformable[d]];
        if (!m.count) continue;
        std::copy(ap.rest.begin(), ap.rest.end(), rest.begin() + (size_t)m.vbase * 8);
        if (m.sets) { std::copy(ap.joints.begin(), ap.joints.end(), joints.begin() + m.jw_base); std::copy(ap.weights.begin(), ap.weights.end(), weights.begin() + m.jw_base); }
        if (m.flags & POSE_GEN_NORMALS) std::copy(ap.last_face.begin(), ap.last_face.end(), last_face.begin() + m.vbase);
        struct { uint32_t flag, c0, nc; const std::vector<float> *src; } planes[3] = { { POSE_DPOS, 0, 3, &ap.dpos }, { POSE_DNRM, 3, 3, &ap.dnrm }, { POSE_DUV, 6, 2, &ap.duv } };
        for (auto &P : planes) if (m.flags & P.flag)
            for (uint32_t t = 0; t < m.targets; t++) for (uint32_t c = 0; c < P.nc; c++) for (uint32_t i = 0; i < m.count; i++)
                deltas[m.delta_base + ((size_t)t * 8 + P.c0 + c) * m.count + i] = (*P.src)[((size_t)t * m.count + i) * P.nc + c];
    }
    auto up = [&](const void *src, size_t bytes) -> void * {
        void *p = pose_blocks_.out<uint8_t>(std::max<size_t>(bytes, 16));
        if (src && bytes) CK(cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice));
        return p;
    };
    pose_dev_.meshes = static_cast<const PoseMesh *>(up(pose_meshes_.data(), pose_meshes_.size() * sizeof(PoseMesh)));
    pose_dev_.block_mesh = static_cast<const uint32_t *>(up(block_mesh.data(), block_mesh.size() * 4));
    pose_dev_.rest = static_cast<const float *>(up(rest.data(), rest.size() * 4));
    pose_dev_.joints = static_cast<const uint32_t *>(up(joints.data(), joints.size() * 4));
    pose_dev_.weights = static_cast<const float *>(up(weights.data(), weights.size() * 4));
    pose_dev_.deltas = static_cast<const float *>(up(deltas.data(), deltas.size() * 4));
    pose_dev_.last_face = static_cast<const uint32_t *>(up(pose_gen_normals_ ? last_face.data() : nullptr, pose_gen_normals_ ? last_face.size() * 4 : 0));
    pose_dev_.indices = d_indices_.get();
    pose_dev_.palette = static_cast<const float *>(up(nullptr, (size_t)pose_palette_floats_ * 4));
    pose_dev_.morph = static_cast<const float *>(up(nullptr, (size_t)pose_morph_floats_ * 4));
    pose_grid_ = (uint32_t)block_mesh.size(); pose_vertices_ = (uint32_t)nv;
}

void Engine::free_pose_data() {
    pose_blocks_.clear(); pose_dev_ = PoseDev{}; pose_meshes_.clear(); pose_grid_ = pose_vertices_ = 0;
}

// glTF pose (DESIGN §15): arguments checked, the waves in flight finished, the pose evaluated on the host (animation.cpp), its joint
// palettes and morph weights uploaded, the deformable meshes' vertices posed from the rest data into the staging buffer and checked there,
// then committed with every instance transform and one refit / rebuild.  A rejected pose changes nothing.
void Engine::pose(int animation, float t, int rebuild) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!scene_.animation) throw CudaError{ B200PT_ERR_NO_SCENE, "the scene has no glTF node data (loaded from OBJ or set through arrays)" };
    if (animation < -1 || animation >= (int)scene_.animation->clips.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "animation index out of range" };
    if (!std::isfinite(t)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "time is not finite" };
    sync_all();
    HostPose P;
    evaluate_pose(*scene_.animation, scene_, animation, t, P);
    std::vector<VertexSource> src;
    if (pose_vertices_) {
        if (P.palette.size() != pose_palette_floats_ || P.morph.size() != pose_morph_floats_) throw CudaError{ B200PT_ERR_UNKNOWN, "pose layout mismatch" };
        b200pt_vertex *stage = static_cast<b200pt_vertex *>(scratch((size_t)pose_vertices_ * sizeof(b200pt_vertex) + 16));
        uint32_t *flag = reinterpret_cast<uint32_t *>(stage + pose_vertices_);
        if (!P.palette.empty()) CK(cudaMemcpyAsync(const_cast<float *>(pose_dev_.palette), P.palette.data(), P.palette.size() * 4, cudaMemcpyHostToDevice, stream_));
        if (!P.morph.empty()) CK(cudaMemcpyAsync(const_cast<float *>(pose_dev_.morph), P.morph.data(), P.morph.size() * 4, cudaMemcpyHostToDevice, stream_));
        CK(cudaMemsetAsync(flag, 0, 4, stream_));
        const int r = launch_pose(pose_dev_, pose_grid_, pose_max_joints_, pose_gen_normals_, stage, flag, stream_);
        if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("launch_pose failed: ") + cudaGetErrorString((cudaError_t)r) };
        CK(cudaMemcpyAsync(h_small_.get(), flag, 4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));                     // also: P's host arrays are no longer read
        if (*h_small_) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "a posed vertex component is not finite" };
        for (size_t d = 0; d < pose_meshes_.size(); d++)
            src.push_back({ (uint32_t)scene_.animation->deformable[d], stage + pose_meshes_[d].vbase, true });
    }
    commit(src, &P.instances, rebuild);
}

// 1x1 textures (the defaults of PathTracer.cpp:1557-1621, or any constant texture) are resolved to their texel value here
DevMaterial Engine::make_dev_material(const b200pt_material &m) const {
    DevMaterial d; memset(&d, 0, sizeof d);
    d.m = m;
    auto texel = [&](uint32_t idx, float4 &out) -> bool {
        if (idx >= scene_.textures.size()) return false;
        const HostTexture &t = scene_.textures[idx];
        if (t.width != 1 || t.height != 1) return false;
        if (t.channels == 4) out = make_float4((float)t.data[0] / 255.0f, (float)t.data[1] / 255.0f, (float)t.data[2] / 255.0f, (float)t.data[3] / 255.0f);
        else out = make_float4((float)t.data[0] / 255.0f, 0.0f, 0.0f, 1.0f);
        return true;
    };
    float4 v;
    if (texel(m.BaseColorTextureIndex, v)) { d.const_mask |= 1u; d.cbase = v; }
    if (texel(m.NormalTextureIndex, v)) { d.const_mask |= 2u; d.cnormal = v; }
    if (texel(m.RoughnessTextureIndex, v)) { d.const_mask |= 4u; d.crough = v.x; }
    if (texel(m.MetallicTextureIndex, v)) { d.const_mask |= 8u; d.cmetal = v.x; }
    if (texel(m.EmissiveTextureIndex, v)) { d.const_mask |= 16u; d.cemis = v; }
    return d;
}

// Shading class of every triangle (device_types.h: MaterialClass): decides the hit queue k_extend appends to and the k_shade_hit<CLASS>
// instantiation that shades it.  Uses the same products the device evaluates (Metallic * texel, material_apply_texels in shading.cuh).
void Engine::rebuild_tri_class() {
    std::vector<uint8_t> cls(scene_.materials.size(), (uint8_t)MC_GENERAL);
    for (size_t i = 0; i < scene_.materials.size(); i++) {
        const DevMaterial dm = make_dev_material(scene_.materials[i]);
        if (!(dm.const_mask & 8u)) continue;                                // metallic texture is not 1x1: the lobe set depends on the texel
        const float metal = dm.m.Metallic * dm.cmetal, T = dm.m.Transmission;
        if (metal == 1.0f) cls[i] = (uint8_t)MC_METAL;
        else if (metal == 0.0f && T == 0.0f) cls[i] = (uint8_t)MC_DIFFUSE;
        else if (metal == 0.0f && T == 1.0f) cls[i] = (uint8_t)MC_GLASS;
    }
    if (const char *e = getenv("B200PT_CLASSES")) { if (atoi(e) == 0) std::fill(cls.begin(), cls.end(), (uint8_t)MC_GENERAL); }   // A/B: one general queue
    std::vector<uint8_t> tc(std::max<size_t>(1, n_tris_), (uint8_t)MC_GENERAL);
    class_mask_ = 0;
    for (size_t i = 0; i < scene_.instances.size(); i++) {
        const uint8_t c = cls[scene_.instances[i].MaterialIndex];
        const uint32_t first = h_instances_[i].tri_base, cnt = h_meshes_[scene_.instances[i].MeshIndex].tri_count;
        if (cnt) { class_mask_ |= 1u << c; std::fill(tc.begin() + first, tc.begin() + first + cnt, c); }
    }
    CK(cudaMemcpy(d_tri_class_.get(), tc.data(), tc.size(), cudaMemcpyHostToDevice));
}

// emissive-mesh list: PathTracer.cpp:458-469 (+ SetMaterial maintenance :712-810); keyed on constant EmissiveColor != 0 (Q16).
// The emissive records, tables and counts change together, after every upload has succeeded; d_instances_ (which carries the counts) is the
// caller's to upload.
void Engine::rebuild_emissive() {
    std::vector<DevEmissive> em;
    for (size_t i = 0; i < scene_.instances.size(); i++) {
        const b200pt_instance &in = scene_.instances[i];
        const b200pt_material &m = scene_.materials[in.MaterialIndex];
        if (m.EmissiveColor[0] != 0.0f || m.EmissiveColor[1] != 0.0f || m.EmissiveColor[2] != 0.0f) {
            DevEmissive e; e.mesh = in.MeshIndex; e.material = in.MaterialIndex; e.tri_count = h_meshes_[in.MeshIndex].tri_count; e.instance = (uint32_t)i;
            memcpy(e.xf, in.Transform, sizeof e.xf);
            em.push_back(e);
        }
    }
    if (em.size() >= 10000) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "too many emissive meshes (MAX_EMISSIVE_MESHES)" };
    // world-space emissive triangles (SH/Sampler.slang:376-391: vertices fetched and transformed per sample in the reference)
    std::vector<EmTri> et; std::vector<uint32_t> base;
    for (const DevEmissive &e : em) {
        base.push_back((uint32_t)et.size());
        const HostMesh &hm = scene_.meshes[e.mesh];
        auto xf = [&](const b200pt_vertex &v) {
            const float *t = e.xf; const float x = v.Position[0], y = v.Position[1], z = v.Position[2];
            return make_float3(t[0] * x + t[4] * y + t[8] * z + t[12] * 1.0f, t[1] * x + t[5] * y + t[9] * z + t[13] * 1.0f, t[2] * x + t[6] * y + t[10] * z + t[14] * 1.0f);
        };
        for (uint32_t t = 0; t < e.tri_count; t++) {
            const b200pt_vertex &A = hm.vertices[hm.indices[t * 3]], &B = hm.vertices[hm.indices[t * 3 + 1]], &C = hm.vertices[hm.indices[t * 3 + 2]];
            const float3 p0 = xf(A), p1 = xf(B), p2 = xf(C);
            EmTri r;
            r.r[0] = make_float4(p0.x, p0.y, p0.z, A.TexCoord[0]); r.r[1] = make_float4(p1.x, p1.y, p1.z, A.TexCoord[1]);
            r.r[2] = make_float4(p2.x, p2.y, p2.z, B.TexCoord[0]);
            const uint32_t gid = h_instances_[e.instance].tri_base + t; float gidf; memcpy(&gidf, &gid, 4);
            r.r[3] = make_float4(B.TexCoord[1], C.TexCoord[0], C.TexCoord[1], gidf);
            et.push_back(r);
        }
    }
    DevPtr<EmTri> em_tris; DevPtr<uint32_t> em_tri_base;
    CK(alloc(em_tris, std::max<size_t>(1, et.size()) * sizeof(EmTri))); CK(alloc(em_tri_base, std::max<size_t>(1, base.size()) * sizeof(uint32_t)));
    if (!et.empty()) CK(cudaMemcpy(em_tris.get(), et.data(), et.size() * sizeof(EmTri), cudaMemcpyHostToDevice));
    if (!base.empty()) CK(cudaMemcpy(em_tri_base.get(), base.data(), base.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    if (!em.empty()) CK(cudaMemcpy(d_emissive_.get(), em.data(), em.size() * sizeof(DevEmissive), cudaMemcpyHostToDevice));
    d_em_tris_ = std::move(em_tris); d_em_tri_base_ = std::move(em_tri_base);
    n_emissive_ = (uint32_t)em.size();
    for (DevInstance &d : h_instances_) d.emissive_tri_count = 0;
    for (const DevEmissive &e : em) h_instances_[e.instance].emissive_tri_count = e.tri_count;
}

void Engine::set_material(uint32_t idx, const b200pt_material &m) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (idx >= scene_.materials.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "material index out of range" };
    const uint32_t tix[5] = { m.BaseColorTextureIndex, m.NormalTextureIndex, m.RoughnessTextureIndex, m.MetallicTextureIndex, m.EmissiveTextureIndex };
    for (uint32_t t : tix) if (t >= scene_.textures.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "texture index out of range" };
    sync_all();
    scene_.materials[idx] = m;
    { const DevMaterial dm = make_dev_material(m); CK(cudaMemcpy(d_materials_.get() + idx, &dm, sizeof dm, cudaMemcpyHostToDevice)); launch_prepare_materials(d_materials_.get(), idx, 1, stream_); CK(cudaStreamSynchronize(stream_)); }
    rebuild_emissive();
    upload_instances();
    rebuild_tri_class();
    reset();
}

// PathTracer::AddVolume / SetVolume / RemoveVolume / AddDensityDataToVolume / RemoveDensityDataFromVolume (PathTracer.cpp:1334-1555)
static void check_volume(const b200pt_volume &v) {
    for (int k = 0; k < 3; k++) if (!(v.CornerMin[k] <= v.CornerMax[k]) || !(v.Scale[k] >= 0.0f)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume AABB: CornerMin > CornerMax or negative Scale" };
    if (!(v.Density >= 0.0f)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume density must be >= 0" };
}
void Engine::upload_volumes() {
    CK(cudaSetDevice(device_));
    sync_all();
    if (!d_volumes_) CK(alloc(d_volumes_, B200PT_MAX_VOLUMES * sizeof(DevVolume)));
    if (!d_grids_) CK(alloc(d_grids_, B200PT_MAX_VOLUMES * sizeof(DevGrid)));
    std::vector<DevVolume> dv(volumes_.size());
    std::vector<DevGrid> dg;
    for (size_t i = 0; i < volumes_.size(); i++) {
        const b200pt_volume &v = volumes_[i];
        float lo[3], hi[3];                                                     // VolumeGPU's constructor, PathTracer.h:396-397
        for (int k = 0; k < 3; k++) { lo[k] = v.Position[k] + (v.CornerMin[k] * v.Scale[k]); hi[k] = v.Position[k] + (v.CornerMax[k] * v.Scale[k]); }
        dv[i].mn_density = make_float4(lo[0], lo[1], lo[2], v.Density);
        dv[i].mx_g = make_float4(hi[0], hi[1], hi[2], v.Anisotropy);
        dv[i].color_alpha = make_float4(v.Color[0], v.Color[1], v.Color[2], v.Alpha);
        dv[i].emis_droplet = make_float4(v.EmissiveColor[0], v.EmissiveColor[1], v.EmissiveColor[2], v.DropletSize);
        dv[i].tcol_gamma = make_float4(v.TemperatureColor[0], v.TemperatureColor[1], v.TemperatureColor[2], v.TemperatureGamma);
        dv[i].tparams = make_float4(v.TemperatureScale, v.EmissiveColorGamma, v.ApproximatedScatteringFalloff, v.GridSharpness);
        dv[i].kelvin = make_float4((float)v.KelvinMin, (float)(v.KelvinMax - v.KelvinMin), v.MaxDensityInTheGrid, 0.0f);
        uint32_t slot = 0xFFFFFFFFu;
        if (grids_[i]) {
            const GridData &G = *grids_[i];
            DevGrid g{};
            g.values = G.d_values.get(); g.max_densities = G.d_max_densities.get();
            for (int k = 0; k < 3; k++) { g.imin[k] = G.host.imin[k]; g.dim[k] = G.host.dim[k]; g.wmin[k] = G.host.wmin[k]; g.wext[k] = G.host.wext[k]; g.inv_vs[k] = G.host.inv_vs[k]; g.trans[k] = G.host.trans[k]; }
            slot = (uint32_t)dg.size(); dg.push_back(g);
        }
        dv[i].flags = make_uint4(v.ApproximatedScatteringForClouds, (uint32_t)(v.HasTemperatureData != 0), (uint32_t)(v.UseBlackbody != 0), slot);
    }
    if (!dv.empty()) CK(cudaMemcpy(d_volumes_.get(), dv.data(), dv.size() * sizeof(DevVolume), cudaMemcpyHostToDevice));
    if (!dg.empty()) CK(cudaMemcpy(d_grids_.get(), dg.data(), dg.size() * sizeof(DevGrid), cudaMemcpyHostToDevice));
    reset();
}
// the three READ-ONLY members of b200pt_volume follow the density data attached to the index, whatever the caller's struct says
static b200pt_volume with_grid_fields(b200pt_volume v, const b200pt_volume *keep) {
    v.DensityDataIndex = keep ? keep->DensityDataIndex : -1;
    v.MaxDensityInTheGrid = keep ? keep->MaxDensityInTheGrid : 0.0f;
    v.HasTemperatureData = keep ? keep->HasTemperatureData : 0;
    return v;
}
uint32_t Engine::add_volume(const b200pt_volume &v) {
    check_volume(v);
    if (volumes_.size() >= B200PT_MAX_VOLUMES) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "too many volumes (B200PT_MAX_VOLUMES)" };
    volumes_.push_back(with_grid_fields(v, nullptr)); grids_.push_back(nullptr); upload_volumes();
    return (uint32_t)volumes_.size() - 1u;
}
void Engine::set_volume(uint32_t idx, const b200pt_volume &v) {
    check_volume(v);
    if (idx >= volumes_.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume index out of range" };
    const b200pt_volume old = volumes_[idx];
    volumes_[idx] = with_grid_fields(v, grids_[idx] ? &old : nullptr); upload_volumes();
}
void Engine::remove_volume(uint32_t idx) {
    if (idx >= volumes_.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume index out of range" };
    sync_all();                                                                 // the grid's device buffers may still be read by waves in flight
    volumes_.erase(volumes_.begin() + idx); grids_.erase(grids_.begin() + idx); upload_volumes();
}
void Engine::add_density_grid(uint32_t idx, const b200pt_density_grid &g) {
    if (idx >= volumes_.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume index out of range" };   // PathTracer.cpp:1348-1352
    auto G = std::make_shared<GridData>();
    prepare_density_grid(g, G->host);
    CK(cudaSetDevice(device_));
    sync_all();
    CK(alloc(G->d_values, G->host.values.size() * sizeof(float)));
    CK(alloc(G->d_max_densities, G->host.max_densities.size() * sizeof(float)));
    CK(cudaMemcpy(G->d_values.get(), G->host.values.data(), G->host.values.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(G->d_max_densities.get(), G->host.max_densities.data(), G->host.max_densities.size() * sizeof(float), cudaMemcpyHostToDevice));
    b200pt_volume &v = volumes_[idx];
    for (int k = 0; k < 3; k++) { v.CornerMin[k] = G->host.corner_min[k]; v.CornerMax[k] = G->host.corner_max[k]; }
    v.MaxDensityInTheGrid = G->host.max_density;
    v.HasTemperatureData = G->host.has_temperature ? 1 : 0;
    v.DensityDataIndex = density_data_counter_;                                 // :1512-1513
    density_data_counter_ = (density_data_counter_ + 1) % (int)B200PT_MAX_VOLUMES;
    grids_[idx] = std::move(G);
    upload_volumes();
}
void Engine::remove_density_data(uint32_t idx) {                                // PathTracer.cpp:1518-1528
    if (idx >= volumes_.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume index out of range" };
    sync_all();
    grids_[idx] = nullptr;
    b200pt_volume &v = volumes_[idx];
    v.DensityDataIndex = -1; v.MaxDensityInTheGrid = 0.0f; v.HasTemperatureData = 0;
    for (int k = 0; k < 3; k++) { v.CornerMin[k] = -1.0f; v.CornerMax[k] = 1.0f; }
    upload_volumes();
}
void Engine::set_phase_function(uint32_t pf) {
    if (pf > 2u) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "phase function: 0 HG, 1 Draine, 2 HG + Draine" };
    phase_function_ = pf; reset();
}

// PathTracer::LoadEnvironmentMap (PathTracer.cpp:1137-1332)
void Engine::set_env_map(uint32_t w, uint32_t h, const float *rgba) {
    CK(cudaSetDevice(device_));
    if (!w || !h || !rgba || (uint64_t)w * h > 0x7FFFFFFFull) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bad environment map" };
    sync_all();
    std::vector<float> px(rgba, rgba + (size_t)w * h * 4);
    std::vector<uint2> alias((size_t)w * h);
    build_env_alias(px.data(), w, h, alias.data());
    // The previous map is released first; the new one is filled in local owners and moved in once every upload has succeeded.
    d_env_.reset(); d_alias_.reset(); d_env_row_cos_.reset();
    DevPtr<float4> d_env; DevPtr<uint2> d_alias; DevPtr<float2> d_row_cos;
    {   // SH/Sampler.slang:329-331: stepTheta = M_PI / height; theta0 = py * stepTheta; cos(theta0), cos(theta0 + stepTheta)
        std::vector<float2> rc(h); const float stepTheta = 3.1415926535897F / (float)h;
        for (uint32_t y = 0; y < h; y++) { const float t0 = (float)y * stepTheta; rc[y] = make_float2(cosf(t0), cosf(t0 + stepTheta)); }
        CK(alloc(d_row_cos, rc.size() * sizeof(float2))); CK(cudaMemcpy(d_row_cos.get(), rc.data(), rc.size() * sizeof(float2), cudaMemcpyHostToDevice));
    }
    CK(alloc(d_env, px.size() * 4)); CK(cudaMemcpy(d_env.get(), px.data(), px.size() * 4, cudaMemcpyHostToDevice));
    CK(alloc(d_alias, alias.size() * sizeof(uint2))); CK(cudaMemcpy(d_alias.get(), alias.data(), alias.size() * sizeof(uint2), cudaMemcpyHostToDevice));
    d_env_ = std::move(d_env); d_alias_ = std::move(d_alias); d_env_row_cos_ = std::move(d_row_cos); env_w_ = w; env_h_ = h;
    reset();
}

void Engine::set_luts(const float *refl, const float *rout, const float *rin) {
    CK(cudaSetDevice(device_));
    if (!refl || !rout || !rin) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "null LUT" };
    sync_all();
    const size_t n[3] = { 64 * 64 * 32, 128 * 128 * 32, 128 * 128 * 32 }; const float *src[3] = { refl, rout, rin };
    // Each previous table is released before its replacement is allocated; the new ones are moved in once every upload has succeeded.
    DevPtr<float> luts[3];
    for (int i = 0; i < 3; i++) { d_luts_[i].reset(); CK(alloc(luts[i], n[i] * 4)); CK(cudaMemcpy(luts[i].get(), src[i], n[i] * 4, cudaMemcpyHostToDevice)); }
    for (int i = 0; i < 3; i++) d_luts_[i] = std::move(luts[i]);
    reset();
}

void Engine::set_config(const b200pt_config &c) {
    if (c.SamplesPerFrame == 0 || c.ScreenChunkCount == 0 || c.ScreenChunkCount > 64) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "SamplesPerFrame and ScreenChunkCount must be >= 1" };
    // The clamp scales a contribution by MaxLuminance / max(lum, MaxLuminance): +inf gives inf / inf = NaN on every segment at Depth != 1, 0 gives
    // 0 / 0 on every zero contribution and NaN gives NaN everywhere, and the sample rejection then discards the whole path (a black image).
    if (!std::isfinite(c.MaxLuminance) || !(c.MaxLuminance > 0.0f)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "MaxLuminance must be finite and > 0" };
    if (c.ScreenChunkCount > 1 && world_ > 1) throw CudaError{ B200PT_ERR_NOT_IMPLEMENTED, "ScreenChunkCount > 1 cannot be combined with a multi-GPU partition" };
    if (c.ScreenChunkCount > 1 && adaptive_.Enable) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "ScreenChunkCount > 1 cannot be combined with adaptive sampling" };
    if (c.ScreenChunkCount > 1 && track_variance_) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "ScreenChunkCount > 1 cannot be combined with per-pixel statistics" };
    cfg_ = c;
    reset();
}

// ---------------------------------------------------------------- adaptive sampling
void Engine::set_adaptive(const b200pt_adaptive &a) {
    if (!std::isfinite(a.Threshold) || a.Threshold < 0.0f) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "adaptive Threshold must be finite and >= 0" };
    if (a.MinSamples < 2 || a.Interval == 0) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "adaptive MinSamples must be >= 2 and Interval >= 1" };
    if (a.Enable && cfg_.ScreenChunkCount > 1) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "adaptive sampling cannot be combined with ScreenChunkCount > 1" };
    CK(cudaSetDevice(device_));
    sync_all();
    adaptive_ = a;
    adaptive_.Enable = a.Enable ? 1u : 0u;
    if (!records()) free_adaptive();
    reset();
}
void Engine::set_track_variance(bool on) {
    if (on && cfg_.ScreenChunkCount > 1) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "per-pixel statistics cannot be combined with ScreenChunkCount > 1" };
    CK(cudaSetDevice(device_));
    sync_all();
    track_variance_ = on;
    if (!records()) free_adaptive();
    reset();
}
void Engine::free_adaptive() {
    d_px_state_.reset(); d_active_.reset(); d_tile_count_.reset(); d_active_count_.reset();
    adaptive_pixels_ = 0; adaptive_ready_ = false;
}
void Engine::update_active(bool decide, cudaStream_t st) {
    const uint32_t npix = (uint32_t)adaptive_pixels_;
    launch_adaptive_update(d_px_state_.get(), npix, adaptive_.Threshold, adaptive_.MinSamples, decide, d_tile_count_.get(), d_active_.get(), d_active_count_.get(), st);
    CK(cudaMemcpyAsync(h_active_count_.get(), d_active_count_.get(), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    active_count_ = *h_active_count_;
}
// After a reset: every local pixel active with an empty record.
void Engine::prepare_adaptive() {
    if (adaptive_ready_) return;
    sync_all();
    const size_t npix = (size_t)W_ * local_rows_;
    if (npix != adaptive_pixels_ || !d_px_state_) {
        free_adaptive();
        const size_t n = std::max<size_t>(npix, 1), tiles = (n + ADAPTIVE_TILE - 1) / ADAPTIVE_TILE;
        CK(alloc(d_px_state_, n * sizeof(uint4))); CK(alloc(d_active_, n * sizeof(uint32_t)));
        CK(alloc(d_tile_count_, tiles * sizeof(uint32_t))); CK(alloc(d_active_count_, sizeof(uint32_t)));
        adaptive_pixels_ = npix;
    }
    CK(cudaMemsetAsync(d_px_state_.get(), 0, std::max<size_t>(npix, 1) * sizeof(uint4), stream_));
    update_active(false, stream_);
    adaptive_ready_ = true;
}
uint32_t Engine::active_pixels() {
    CK(cudaSetDevice(device_));
    if (!adaptive_.Enable) return W_ * local_rows_;
    if (!adaptive_ready_) { if (!has_scene_ || !W_) return W_ * local_rows_; prepare_adaptive(); }
    return active_count_;
}
void Engine::pixel_stats(uint32_t *counts, float *rel_error) {
    CK(cudaSetDevice(device_));
    const size_t npix = (size_t)W_ * local_rows_;
    if (!records() || !adaptive_ready_) {
        if (counts) std::fill(counts, counts + npix, frame_count_);
        if (rel_error) std::fill(rel_error, rel_error + npix, std::nanf(""));
        return;
    }
    sync_all();
    std::vector<uint4> st(npix);
    CK(cudaMemcpy(st.data(), d_px_state_.get(), npix * sizeof(uint4), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < npix; i++) {
        const uint32_t n = st[i].z;
        if (counts) counts[i] = n;
        if (rel_error) {
            float meanL, M2; memcpy(&meanL, &st[i].x, 4); memcpy(&M2, &st[i].y, 4);
            rel_error[i] = n < 2 ? std::nanf("") : (float)(std::sqrt((double)M2 / (double)(n - 1) / (double)n) / std::max((double)meanL, 1e-3));
        }
    }
}
void Engine::set_camera(const float vi[16], const float pi[16]) { memcpy(view_inv_, vi, sizeof view_inv_); memcpy(proj_inv_, pi, sizeof proj_inv_); reset(); }
void Engine::get_camera(float vi[16], float pi[16]) const { memcpy(vi, view_inv_, sizeof view_inv_); memcpy(pi, proj_inv_, sizeof proj_inv_); }
void Engine::reset() { dispatch_count_ = 0; frame_count_ = 0; samples_accumulated_ = 0; adaptive_ready_ = false; }   // PathTracer.h:183

void Engine::resize(uint32_t w, uint32_t h) {                                                  // PathTracer::ResizeImage
    if (!w || !h || w > 65535 || h > 65535) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bad image size" };
    CK(cudaSetDevice(device_));
    sync_all();
    W_ = w; H_ = h; local_rows_ = partition_local_rows(H_, rank_, world_, band_);
    ensure_image(); reset();
}
void Engine::set_partition(uint32_t rank, uint32_t world, uint32_t band) {
    if (!world || rank >= world || !band) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bad partition" };
    if (world > 1 && cfg_.ScreenChunkCount > 1) throw CudaError{ B200PT_ERR_NOT_IMPLEMENTED, "ScreenChunkCount > 1 cannot be combined with a multi-GPU partition" };
    CK(cudaSetDevice(device_));
    sync_all();
    rank_ = rank; world_ = world; band_ = band;
    if (W_ && H_) { local_rows_ = partition_local_rows(H_, rank_, world_, band_); ensure_image(); }
    reset();
}
void Engine::ensure_image() {
    const size_t need = (size_t)W_ * std::max<uint32_t>(local_rows_, 1);
    if (need != image_pixels_) { CK(alloc(d_image_, need * sizeof(float4))); image_pixels_ = need; }
    CK(cudaMemsetAsync(d_image_.get(), 0, image_pixels_ * sizeof(float4), stream_));
}

void Engine::free_wave() {
    for (auto &B : wb_) {
        B.arrays.clear();
        B.ps[0] = B.ps[1] = PathState{}; B.so = ShadeOut{}; B.sample_buf = nullptr; B.rng_carry = B.q_hit = B.q_miss = nullptr;
        B.cap = 0;
    }
    wave_cap_ = 0;
}
void Engine::ensure_wave(size_t cap, int contexts) {
    bool ok = cap <= wave_cap_;
    for (int c = 0; c < contexts; c++) ok = ok && wb_[c].cap >= cap;
    if (ok) return;
    sync_all();
    cap = std::max(cap, wave_cap_);
    free_wave();
    for (int c = 0; c < contexts; c++) {
        WaveBuf &B = wb_[c];
        auto a4 = [&](float4 *&p) { p = B.arrays.out<float4>(cap); };
        for (auto &p : B.ps) { a4(p.org_pdf); a4(p.dir_rng); a4(p.thr_depth); a4(p.rad_slot); a4(p.medium); p.medium_g = B.arrays.out<float>(cap); p.vol_depth = B.arrays.out<uint32_t>(cap); }
        a4(B.so.hit); a4(B.so.bxdf_pdf); a4(B.so.e0); a4(B.so.sky_o); a4(B.so.sky_d); a4(B.so.sky_c); a4(B.so.lit_o); a4(B.so.lit_d); a4(B.so.lit_c);
        a4(B.sample_buf);
        B.rng_carry = B.arrays.out<uint32_t>(cap);
        B.q_hit = B.arrays.out<uint32_t>((size_t)MC_COUNT * cap); B.q_miss = B.arrays.out<uint32_t>(cap);   // one hit queue per material class
        B.cap = cap;
    }
    wave_cap_ = cap;
}

DevScene Engine::dev_scene() const {
    DevScene sc{};
    sc.verts = d_verts_.get(); sc.indices = d_indices_.get(); sc.meshes = d_meshes_.get(); sc.instances = d_instances_.get();
    sc.materials = d_materials_.get(); sc.textures = d_textures_.get(); sc.tri_class = d_tri_class_.get();
    sc.uniform_class = 0xFFu;
    for (uint32_t c = 0; c < MC_COUNT; c++) if (class_mask_ == (1u << c)) sc.uniform_class = c;
    sc.emissive = d_emissive_.get(); sc.em_tris = d_em_tris_.get(); sc.em_tri_base = d_em_tri_base_.get(); sc.n_emissive = n_emissive_;
    tree_.view(sc);
    sc.env = d_env_.get(); sc.alias = d_alias_.get(); sc.env_row_cos = d_env_row_cos_.get(); sc.envW = env_w_; sc.envH = env_h_;
    sc.lut_reflect = d_luts_[0].get(); sc.lut_refract_out = d_luts_[1].get(); sc.lut_refract_in = d_luts_[2].get();
    if (d_volumes_ && d_grids_) {                       // both allocated by the first upload_volumes
        sc.volumes = d_volumes_.get(); sc.n_volumes = (uint32_t)volumes_.size();
        sc.grids = d_grids_.get(); sc.n_grids = (uint32_t)std::count_if(grids_.begin(), grids_.end(), [](const auto &g) { return g != nullptr; });
    }
    sc.phase_function = phase_function_;
    return sc;
}

DevConfig Engine::make_dev_config() const {
    DevConfig d; memset(&d, 0, sizeof d);
    memcpy(d.VI, view_inv_, sizeof d.VI); memcpy(d.PI, proj_inv_, sizeof d.PI);
    d.SampleCount = cfg_.SamplesPerFrame; d.MaxDepth = cfg_.MaxDepth; d.MaxLuminance = cfg_.MaxLuminance; d.FocusDistance = cfg_.FocusDistance;
    d.DepthOfFieldStrength = cfg_.DepthOfFieldStrength; d.SkyRotationAzimuth = cfg_.SkyRotationAzimuth; d.SkyRotationAltitude = cfg_.SkyRotationAltitude;
    d.EnvironmentIntensity = cfg_.SkyIntensity; d.EmissiveMeshSamplingPDFBias = cfg_.EmissiveMeshSamplingPDFBias; d.ScreenSplitCount = cfg_.ScreenChunkCount;
    d.EnableSkyMIS = cfg_.EnableSkyMIS; d.EnableMeshMIS = cfg_.EnableMeshMIS; d.ShowEnvMapDirectly = cfg_.ShowEnvMapDirectly;
    d.UseOnlyGeometryNormals = cfg_.UseOnlyGeometryNormals; d.UseEnergyCompensation = cfg_.UseEnergyCompensation; d.FurnaceTestMode = cfg_.FurnaceTestMode;
    {   // atmosphere block (PathTracer.h:221-232 -> SH/Bindings.slang:26-37)
        const b200pt_atmosphere &a = atmosphere_;
        d.EnableAtmosphere = a.Enable ? 1u : 0u; d.PlanetRadius = a.PlanetRadius; d.AtmosphereHeight = a.AtmosphereHeight;
        for (int k = 0; k < 3; k++) { d.PlanetPosition[k] = a.PlanetPosition[k]; d.RayleighMult[k] = a.RayleighScatteringCoefficientMultiplier[k]; d.MieMult[k] = a.MieScatteringCoefficientMultiplier[k];
                                      d.OzoneMult[k] = a.OzoneAbsorptionCoefficientMultiplier[k]; d.SunColor[k] = a.SunColor[k]; }
        d.RayleighDensityFalloff = a.RayleighDensityFalloff; d.MieDensityFalloff = a.MieDensityFalloff; d.OzoneDensityFalloff = a.OzoneDensityFalloff; d.OzonePeak = a.OzonePeak;
        d.cosSunTheta = cosf(0.004675f);
    }
    { const float az = cfg_.SkyRotationAzimuth / 180.0f * 3.1415926535897F, al = cfg_.SkyRotationAltitude / 180.0f * 3.1415926535897F;   // SH/Sampler.slang:338-339
      d.cosAz = cosf(az); d.sinAz = sinf(az); d.cosAl = cosf(al); d.sinAl = sinf(al); }
    d.W = W_; d.H = H_; d.rank = rank_; d.world = world_; d.band_rows = band_; d.local_rows = local_rows_;
    return d;
}

// Conservative: the device-side metallic value is Metallic * texel, so the constant factor alone cannot rule refraction out, and a negative
// density (not validated by the reference either) scatters on every segment.  A false positive only costs a 4-byte read-back per 16 bounces.
bool Engine::scene_has_media() const {
    for (const auto &m : scene_.materials) if (m.Transmission > 0.0f && m.MediumDensity != 0.0f && m.MediumAnisotropy != 1.0f) return true;
    return false;
}

// One bounce of path_trace's loop; bounce_query runs the same sequence on caller-given paths.
uint64_t Engine::bounce(const CallPlan &cp, const DevScene &sc, const DevConfig &dc, WaveBuf &B, const PathState pst[2], int cur, uint32_t k, uint32_t flags, cudaStream_t st,
                        const std::function<void(int)> &mark) {
    const uint32_t par = k & 1u;
    const Queues q{ B.q_miss, B.q_hit, (uint32_t)wave_cap_ };
    uint64_t launches = 0;
    if (cp.pre) launches += launch_volume_decide(tree_.lc, sc, dc, pst[cur], B.so, B.counts.get(), par, B.sample_buf, B.rng_carry, st);
    if (!(cp.camera && k == 0)) launches += launch_extend(tree_.lc, cp, sc, pst[cur], B.so.hit, B.counts.get(), par, q, d_ctr_.get(), k == 0, st); mark(1);
    launches += launch_shade(tree_.lc, cp, sc, dc, pst[cur], pst[cur ^ 1], B.so, B.so.hit, B.counts.get(), par, q, B.sample_buf, B.rng_carry, d_ctr_.get(), flags, st); mark(2);
    if (!cp.fuse) launches += launch_connect(tree_.lc, cp, sc, dc, pst[cur], pst[cur ^ 1], B.so, B.counts.get(), par, q, B.sample_buf, B.rng_carry, d_ctr_.get(), flags, st); mark(3);
    return launches;
}

// PathTracer::PathTrace x dispatches (PathTracer.cpp:122-156)
bool Engine::path_trace(uint32_t dispatches, uint32_t base_seed) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "PathTrace before SetScene" };
    if (!has_env()) throw CudaError{ B200PT_ERR_NO_SCENE, "no environment map (PathTracer always loads one, PathTracer.cpp:202)" };
    if (!has_luts()) throw CudaError{ B200PT_ERR_NO_SCENE, "no energy-compensation lookup tables (PathTracer.cpp:199-201)" };
    const uint32_t S = cfg_.ScreenChunkCount, S2 = S * S;
    const bool adaptive = adaptive_.Enable != 0u;              // S == 1 (set_config / set_adaptive / set_track_variance)
    const bool tracked = records();                           // statistics without adaptive sampling: the records over the identity list, no decisions
    if (tracked) prepare_adaptive();
    if (adaptive && active_count_ == 0) return true;          // every local pixel has converged: nothing to launch, the dispatch counter stays
    // how many dispatches until MaxSamplesAccumulated (PathTracer.cpp:124-125,151-153)
    uint32_t todo = 0;
    { uint64_t d = dispatch_count_; uint32_t acc = samples_accumulated_;
      while (todo < dispatches && acc < cfg_.MaxSamplesAccumulated) { d++; todo++; acc = (uint32_t)(d / S2) * cfg_.SamplesPerFrame; } }
    if (todo == 0) return samples_accumulated_ >= cfg_.MaxSamplesAccumulated;
    if (todo > kMaxDispatchTable) todo = kMaxDispatchTable;

    const uint32_t P = (S == 1) ? W_ * local_rows_ : ((W_ + S - 1) / S) * ((H_ + S - 1) / S);
    if (P == 0) { dispatch_count_ += todo; frame_count_ = (uint32_t)(dispatch_count_ / S2); samples_accumulated_ = frame_count_ * cfg_.SamplesPerFrame; return samples_accumulated_ >= cfg_.MaxSamplesAccumulated; }
    // Two waves in flight (two contexts, two internal streams): the late bounces of a wave are bound by the latency chain of their longest rays (a latency floor
    // per traversal launch on large scenes), during which most SMs idle -- the next wave's full-machine bounces fill them.  Waves are
    // numbered across calls (wave_seq_): wave w runs in context w & 1 on internal stream w & 1 and its k_resolve waits for wave w - 1's, so the running mean folds
    // the frames in dispatch order whatever overlaps.  The join with the caller's stream is LAZY: path_trace returns with the waves in flight, and whatever touches
    // the image afterwards (get_hdr, post_process, set_hdr, checkpoints, ...) first makes the caller's stream wait for the resolves (join_waves); the next call's
    // resolves in turn wait for what the caller enqueued on the image in between (image_free_ev_).  So consecutive path_trace calls -- the steps of a multi-GPU
    // run, each followed by an NCCL gather of the bands -- overlap as well: the gather of step k runs beside the first bounces of step k + 1.
    // B200PT_OVERLAP=0 runs one wave at a time on the caller's stream (also used while profiling per-kernel times).
    bool overlap = !profiling_;
    if (const char *e = getenv("B200PT_OVERLAP")) { if (atoi(e) == 0) overlap = false; }
    uint64_t target = 0;                                      // auto wave size (paths per context), when FramesInFlight == 0
    if (cfg_.FramesInFlight == 0) {
        // Auto wave size: up to 64 M paths per context (~24 GB of wavefront state at ~360 B per path; all contexts capped to a quarter of the free HBM): large enough
        // to amortise the floors above.  On an 80 GB H100 the quarter of free HBM, not the 64 M cap, sets the size.
        target = 64ull << 20;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
            uint64_t have = 0; for (const auto &B : wb_) have += (uint64_t)B.cap * 400ull;       // what this engine already holds counts as available
            target = std::min<uint64_t>(target, std::max<uint64_t>(1ull << 20, ((uint64_t)free_b + have) / 4ull / 400ull / (overlap ? 2ull : 1ull)));
        }
    }
    // frames per wave for `frames` frames of P paths each, at most `cap_frames`
    auto wave_frames = [&](uint32_t frames, uint32_t Pw, uint32_t cap_frames) {
        uint32_t F = cfg_.FramesInFlight;
        if (F == 0) F = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(256, target / Pw));
        F = std::max(1u, std::min({ F, frames, cap_frames }));
        const uint32_t n_waves = (frames + F - 1) / F; return (frames + n_waves - 1) / n_waves;   // equal waves: 128 frames at F = 123 become 64 + 64, not 123 + 5
    };
    const uint32_t F = wave_frames(todo, P, todo);
    const int n_ctx = overlap ? 2 : 1;
    ensure_wave((size_t)F * P, n_ctx);                        // adaptive: A <= P, so F * P is the worst case of every interval's waves too
    if (!overlap) join_waves();                               // single-stream mode runs on the caller's stream, behind whatever the internal streams still hold
    else CK(cudaEventRecord(image_free_ev_.get(), stream_));        // what the caller has enqueued on the image so far (gather copy, post chain, set_hdr) precedes this call's resolves
    const DevConfig dc = make_dev_config();
    auto pcg = [](uint32_t in) { uint32_t st = in * 747796405u + 2891336453u; uint32_t w = ((st >> ((st >> 28u) + 4u)) ^ st) * 277803737u; return (w >> 22u) ^ w; };

    const bool medium = scene_has_media();
    DevScene sc = dev_scene();
    const CallPlan cp = plan_call(tree_.lc, sc, dc, medium, class_mask_);
    sc.pre_pass = cp.pre ? 1u : 0u;
    const uint32_t implied_flag = cp.implied ? WAVE_IMPLIED : 0u;   // per-launch flags: kernels.h
    const uint32_t qcap = (uint32_t)wave_cap_;

    uint64_t launches = 0; uint32_t waves = 0, bounces_total = 0;
    std::vector<int> prof_kind; size_t prof_n = 0;            // kind: 0 raygen 1 extend 2 shade 3 connect 4 resolve
    const std::function<void(int)> mark = [&](int kind) {
        if (!profiling_) return;
        if (prof_n >= prof_ev_.size()) prof_ev_.push_back(make_event(cudaEventDefault));
        CK(cudaEventRecord(prof_ev_[prof_n++].get(), stream_)); prof_kind.push_back(kind);
    };
    mark(-1);
    cudaStream_t last_st = stream_;
    // Adaptive sampling cuts the frames into intervals: the waves of an interval trace the A pixels still active (P = A), and at the
    // interval's end k_adaptive_update runs behind the last resolve and A is read back (one host sync per interval).
    for (uint32_t s0 = 0; s0 < todo;) {
        uint32_t seg = todo - s0, Pw = P, Fw = F;
        const uint32_t *const act = adaptive ? d_active_.get() : nullptr;
        if (adaptive) {
            seg = (uint32_t)std::min<uint64_t>(seg, adaptive_.Interval - (dispatch_count_ + s0) % adaptive_.Interval);
            Pw = active_count_;
            Fw = wave_frames(seg, Pw, (uint32_t)std::min<size_t>(wave_cap_ / Pw, 1u << 30));
        }
        for (uint32_t w0 = s0; w0 < s0 + seg; w0 += Fw) {
            const uint32_t nd = std::min(Fw, s0 + seg - w0);
            const int ctx = overlap ? (int)(wave_seq_ & 1ull) : 0;
            WaveBuf &B = wb_[ctx];
            cudaStream_t st = overlap ? aux_stream_[ctx].get() : stream_;
            if (w0 == 0) CK(cudaEventRecord(ev_[0].get(), st));
            // this wave's slice of the dispatch table (PathTracer.cpp:127-150: FrameCount, Seed = PCG(seed + dispatch), ChunkIndex) travels on the wave's own stream
            CK(cudaEventSynchronize(B.disp_ev.get()));                  // the pinned copy is reusable once ITS last upload has executed
            for (uint32_t i = 0; i < nd; i++) {
                const uint64_t d = dispatch_count_ + w0 + i;
                DevDispatch &hd = B.h_disp.get()[i];
                hd.FrameCount = (uint32_t)(d / S2); hd.Seed = pcg(base_seed + (uint32_t)d); hd.ChunkIndex = (uint32_t)(d % S2); hd._pad = 0;
            }
            CK(cudaMemcpyAsync(B.d_disp.get(), B.h_disp.get(), nd * sizeof(DevDispatch), cudaMemcpyHostToDevice, st));
            CK(cudaEventRecord(B.disp_ev.get(), st));
            PathState pst[2] = { B.ps[0], B.ps[1] };              // payload.VolumeDepth travels only while the scene has volumes
            if (!sc.n_volumes) { pst[0].vol_depth = nullptr; pst[1].vol_depth = nullptr; }
            const Queues q{ B.q_miss, B.q_hit, qcap };
            for (uint32_t s = 0; s < cfg_.SamplesPerFrame; s++) {
                const uint32_t wflags = (s == 0 && cp.store ? WAVE_STORE : 0u) | (s + 1 < cfg_.SamplesPerFrame ? WAVE_CARRY : 0u);
                if (cp.camera) {
                    CK(cudaMemsetAsync(B.counts.get(), 0, CTRL_WORDS * sizeof(uint32_t), st));   // before any CTA appends to the parity-0 queues
                    launches += launch_camera(tree_.lc, cp, sc, dc, B.d_disp.get(), nd, Pw, s == 0 ? 1u : 0u, wflags | implied_flag, B.rng_carry, pst[0], B.sample_buf, B.so.hit,
                                              B.counts.get(), q, d_ctr_.get(), st, act);
                } else launches += launch_raygen(tree_.lc, dc, B.d_disp.get(), nd, Pw, s == 0 ? 1u : 0u, wflags, B.rng_carry, pst[0], B.sample_buf, B.counts.get(), d_ctr_.get(), st, act);
                mark(0);
                int cur = 0; uint32_t k = 0;
                for (;;) {
                    uint32_t chunk = 16;
                    if (!medium && cfg_.MaxDepth - std::min(cfg_.MaxDepth, k) < chunk) chunk = cfg_.MaxDepth - std::min(cfg_.MaxDepth, k);
                    if (chunk == 0) break;
                    for (uint32_t b = 0; b < chunk; b++, k++) {
                        launches += bounce(cp, sc, dc, B, pst, cur, k, wflags | (k == 0 ? implied_flag : 0u), st, mark);
                        cur ^= 1;
                    }
                    if (!medium && k >= cfg_.MaxDepth) break;    // every surviving path has Depth >= MaxDepth: provably empty
                    CK(cudaMemcpyAsync(B.h_count.get(), B.counts.get() + (k & 1u), sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
                    CK(cudaStreamSynchronize(st));
                    if (*B.h_count == 0) break;
                    if (k > (1u << 20)) break;                    // runaway guard
                }
                bounces_total += k;
            }
            // the running mean folds the waves in dispatch order: this wave's resolve waits for the previous wave's (the other stream, possibly an earlier call)
            // and for whatever the caller enqueued on the image before this call
            if (overlap) {
                if (wave_seq_ > 0) CK(cudaStreamWaitEvent(st, resolved_ev_[ctx ^ 1].get(), 0));
                CK(cudaStreamWaitEvent(st, image_free_ev_.get(), 0));
            }
            if (tracked) launch_resolve_adaptive(tree_.lc, dc, nd, Pw, d_active_.get(), B.sample_buf, d_image_.get(), d_px_state_.get(), st);
            else launch_resolve(tree_.lc, dc, B.d_disp.get(), nd, P, B.sample_buf, d_image_.get(), st);
            CK(cudaEventRecord(resolved_ev_[ctx].get(), st));
            wave_seq_++;
            launches++; waves++; mark(4);
            last_st = st;
        }
        s0 += seg;
        if (adaptive && (dispatch_count_ + s0) % adaptive_.Interval == 0) {
            // the last resolve of the interval follows every earlier wave's resolve (and so every camera kernel that read the list)
            update_active(true, last_st);
            launches += 2;
            if (active_count_ == 0) { todo = s0; break; }     // the frames not traced do not count
        }
    }
    CK(cudaEventRecord(ev_[1].get(), last_st));                     // ms_total: first kernel of the first wave .. resolve of the last (counters() synchronises before reading it)
    timed_ = true;
    CK(cudaGetLastError());
    dispatch_count_ += todo;
    frame_count_ = (uint32_t)(dispatch_count_ / S2);                     // PathTracer.cpp:152
    samples_accumulated_ = frame_count_ * cfg_.SamplesPerFrame;          // :153
    last_.kernel_launches += launches; last_.waves = waves; last_.bounces = bounces_total;
    last_.ms_raygen = last_.ms_extend = last_.ms_shade = last_.ms_connect = last_.ms_resolve = 0.0f;
    if (profiling_ && prof_n > 1) {
        CK(cudaStreamSynchronize(stream_));
        float *acc[5] = { &last_.ms_raygen, &last_.ms_extend, &last_.ms_shade, &last_.ms_connect, &last_.ms_resolve };
        for (size_t i = 1; i < prof_n; i++) { float ms = 0.0f; CK(cudaEventElapsedTime(&ms, prof_ev_[i - 1].get(), prof_ev_[i].get())); if (prof_kind[i] >= 0) *acc[prof_kind[i]] += ms; }
    }
    return samples_accumulated_ >= cfg_.MaxSamplesAccumulated || (adaptive && active_count_ == 0);
}

void Engine::set_stream(cudaStream_t s) {
    CK(cudaSetDevice(device_));
    sync_all();
    stream_ = s ? s : own_stream_.get();
}

void Engine::synchronize() { CK(cudaSetDevice(device_)); sync_all(); CK(cudaGetLastError()); }

b200pt_counters Engine::counters() {
    CK(cudaSetDevice(device_));
    sync_all();
    WaveCounters wc; CK(cudaMemcpy(&wc, d_ctr_.get(), sizeof wc, cudaMemcpyDeviceToHost));
    b200pt_counters c = last_;
    c.paths = wc.paths; c.extend_rays = wc.extend_rays; c.shade_invocations = wc.shade_invocations; c.surface_hits = wc.surface_hits;
    c.misses = wc.misses; c.shadow_rays = wc.shadow_rays; c.medium_events = wc.medium_events;
    float ms = 0.0f;
    if (timed_) CK(cudaEventElapsedTime(&ms, ev_[0].get(), ev_[1].get()));   // (querying never-recorded events would leave an error for the next call to find)
    c.ms_total = ms;
    return c;
}

void Engine::get_hdr(float *dst, bool dev) {
    CK(cudaSetDevice(device_));
    if (!d_image_ || !dst) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "no image" };
    join_waves();
    CK(cudaMemcpyAsync(dst, d_image_.get(), (size_t)W_ * local_rows_ * sizeof(float4), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream_));
    if (!dev) CK(cudaStreamSynchronize(stream_));        // a device destination stays asynchronous on the engine's stream: the NCCL gather that follows is stream-ordered,
                                                          // and the host can already enqueue the next wave (no per-step bubble on multi-GPU runs)
}
void Engine::set_hdr(const float *src, bool dev) {
    CK(cudaSetDevice(device_));
    if (!d_image_ || !src) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "no image" };
    join_waves();
    CK(cudaMemcpyAsync(d_image_.get(), src, (size_t)W_ * local_rows_ * sizeof(float4), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, stream_));
    CK(cudaStreamSynchronize(stream_));
}

// ---------------------------------------------------------------- checkpoint / resume
// The whole progressive state of the reference is the RGBA32F image + three counters (PT/PathTracer.h:199-201); frame f always uses
// Seed_f = PCG(base_seed + dispatch index), so a render resumed from a checkpoint continues the SAME sample sequence: N frames in one go
// and k frames + checkpoint + (N - k) frames give bit-identical images (tested).  File: 64-byte header + local rows of float4; version 2
// (adaptive sampling or per-pixel statistics on) appends the 16-byte b200pt_adaptive block and one 16-byte record per local pixel.
namespace {
struct CkptHeader { char magic[8]; uint32_t version, W, H, rank, world, band, local_rows, frame_count, samples_accumulated, samples_per_frame, chunk_count, _pad; uint64_t dispatch_count; };
static_assert(sizeof(CkptHeader) == 64, "checkpoint header is 64 B");
}
void Engine::save_checkpoint(const char *path) {
    CK(cudaSetDevice(device_));
    if (!d_image_ || !path) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "no image to checkpoint" };
    std::vector<float> img((size_t)W_ * local_rows_ * 4);
    get_hdr(img.data(), false);
    const bool adaptive = records();
    std::vector<uint4> px;                                    // version 2 (adaptive sampling or statistics on): + the adaptive block + one 16-B record per local pixel
    if (adaptive) {
        prepare_adaptive();
        px.resize((size_t)W_ * local_rows_);
        CK(cudaMemcpy(px.data(), d_px_state_.get(), px.size() * sizeof(uint4), cudaMemcpyDeviceToHost));
    }
    CkptHeader h{}; memcpy(h.magic, "B2PTCKPT", 8); h.version = adaptive ? 2 : 1; h.W = W_; h.H = H_; h.rank = rank_; h.world = world_; h.band = band_; h.local_rows = local_rows_;
    h.frame_count = frame_count_; h.samples_accumulated = samples_accumulated_; h.samples_per_frame = cfg_.SamplesPerFrame; h.chunk_count = cfg_.ScreenChunkCount;
    h.dispatch_count = dispatch_count_;
    FILE *f = fopen(path, "wb");
    if (!f) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, std::string("cannot open checkpoint for writing: ") + path };
    bool ok = fwrite(&h, sizeof h, 1, f) == 1 && fwrite(img.data(), sizeof(float), img.size(), f) == img.size();
    if (ok && adaptive) ok = fwrite(&adaptive_, sizeof adaptive_, 1, f) == 1 && fwrite(px.data(), sizeof(uint4), px.size(), f) == px.size();
    if (fclose(f) != 0 || !ok) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "short write of the checkpoint" };
}
void Engine::load_checkpoint(const char *path) {
    CK(cudaSetDevice(device_));
    if (!d_image_ || !path) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "resize the image before loading a checkpoint" };
    FILE *f = fopen(path, "rb");
    if (!f) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, std::string("cannot open checkpoint: ") + path };
    CkptHeader h{};
    std::vector<float> img;
    bool ok = fread(&h, sizeof h, 1, f) == 1 && memcmp(h.magic, "B2PTCKPT", 8) == 0 && (h.version == 1 || h.version == 2);
    const bool fits = ok && h.W == W_ && h.H == H_ && h.rank == rank_ && h.world == world_ && h.band == band_ && h.local_rows == local_rows_ &&
                      h.samples_per_frame == cfg_.SamplesPerFrame && h.chunk_count == cfg_.ScreenChunkCount;
    if (fits) { img.resize((size_t)W_ * local_rows_ * 4); ok = fread(img.data(), sizeof(float), img.size(), f) == img.size(); }
    // version 2 (adaptive sampling or statistics): the adaptive block must equal this handle's; version 1 cannot resume a render with records
    b200pt_adaptive blk{}; std::vector<uint4> px;
    bool same_mode = h.version == (records() ? 2u : 1u);
    if (fits && ok && same_mode && h.version == 2) {
        ok = fread(&blk, sizeof blk, 1, f) == 1;
        same_mode = ok && memcmp(&blk, &adaptive_, sizeof blk) == 0;
        if (same_mode) { px.resize((size_t)W_ * local_rows_); ok = fread(px.data(), sizeof(uint4), px.size(), f) == px.size(); }
    }
    fclose(f);
    if (!ok) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "not a b200pt checkpoint (bad magic / version / truncated)" };
    if (!fits) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "checkpoint was taken with another image size, partition, SamplesPerFrame or ScreenChunkCount" };
    if (!same_mode) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "checkpoint was taken with other adaptive-sampling or statistics settings" };
    set_hdr(img.data(), false);
    if (records()) {                                   // the records, then the active list rebuilt from their flags
        reset(); prepare_adaptive();
        CK(cudaMemcpy(d_px_state_.get(), px.data(), px.size() * sizeof(uint4), cudaMemcpyHostToDevice));
        update_active(false, stream_);
    }
    dispatch_count_ = h.dispatch_count; frame_count_ = h.frame_count; samples_accumulated_ = h.samples_accumulated;
}

// ---------------------------------------------------------------- PostProcessor (PostProcessor.cpp:128-246)
void Engine::free_post() { d_mips_.clear(); mip_wh_.clear(); d_ldr_.reset(); post_w_ = post_h_ = 0; }
void Engine::ensure_post() {
    if (post_w_ == W_ && post_h_ == H_ && !d_mips_.empty()) return;
    free_post();
    uint32_t wh[20]; const uint32_t levels = bloom_mip_sizes(W_, H_, wh);                     // SetInputImage :128-158
    for (uint32_t i = 0; i < levels; i++) { DevPtr<float4> p; CK(alloc(p, (size_t)wh[2 * i] * wh[2 * i + 1] * sizeof(float4))); d_mips_.push_back(std::move(p)); mip_wh_.push_back(wh[2 * i]); mip_wh_.push_back(wh[2 * i + 1]); }
    CK(alloc(d_ldr_, (size_t)W_ * H_ * sizeof(uchar4)));
    post_w_ = W_; post_h_ = H_;
}
void Engine::accumulate_rows(const float4 *d_frame, uint32_t frame_index, uint32_t y0, uint32_t y1) {
    CK(cudaSetDevice(device_));
    if (!d_image_ || !d_frame || y0 >= y1 || y1 > H_ || world_ != 1) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "accumulate_rows: no image / bad rows / partitioned image" };
    join_waves();
    launch_accumulate(d_frame, d_image_.get(), y0 * W_, (y1 - y0) * W_, frame_index, tree_.lc.grid_light > 0 ? tree_.lc.grid_light : 1184, stream_);
    CK(cudaGetLastError());
}
// HDR rows read by post_process_rows(y0, y1): the final kernel's rows y0-1 .. y1-1 and the first down pass's taps 2y-2 .. 2y+1 over D[1]
void Engine::post_input_rows(uint32_t y0, uint32_t y1, uint32_t *in0, uint32_t *in1) {
    if (y0 >= y1 || y1 > H_) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "post_input_rows: bad row range" };
    ensure_post();
    const uint32_t levels = (uint32_t)d_mips_.size(), mips = std::min(std::max(bloom_.MipCount, 1u), levels);
    int lo = std::max((int)y0 - 1, 0), hi = (int)y1 - 1;
    if (mips >= 2) {
        int U[24][2], D[24][2];
        auto clampr = [&](int v, uint32_t i) { return std::min(std::max(v, 0), (int)mip_wh_[2 * i + 1] - 1); };
        U[1][0] = clampr(lo / 2 - 1, 1); U[1][1] = clampr(hi / 2 + 2, 1);
        for (uint32_t i = 2; i < mips; i++) { U[i][0] = clampr(U[i - 1][0] / 2 - 1, i); U[i][1] = clampr(U[i - 1][1] / 2 + 2, i); }
        D[mips - 1][0] = U[mips - 1][0]; D[mips - 1][1] = U[mips - 1][1];
        for (uint32_t i = mips - 1; i-- > 1;) { D[i][0] = std::min(U[i][0], clampr(2 * D[i + 1][0] - 2, i)); D[i][1] = std::max(U[i][1], clampr(2 * D[i + 1][1] + 1, i)); }
        lo = std::min(lo, std::max(2 * D[1][0] - 2, 0)); hi = std::max(hi, std::min(2 * D[1][1] + 1, (int)H_ - 1));
    }
    *in0 = (uint32_t)lo; *in1 = (uint32_t)hi + 1u;
}
void Engine::post_process() { post_process_rows(0, H_); }

// Row-block post pass (BASELINE config 5 on 2 / 4 / 8 GPUs): rank r holds the full HDR image and produces output rows [y0, y1) only.  The bloom chain is
// evaluated on exactly the rows those outputs depend on -- per mip i the rows U[i] whose post-up value is read and the rows D[i] whose down
// result is read (U[i] plus the taps of the next down pass) -- so the block equals the same rows of the full-image pass bit for bit (tested)
// without any exchange: the halo is recomputed, ~4 rows per level next to a block of H / (N 2^i) rows, the whole mip once it is a few rows tall.
void Engine::post_process_rows(uint32_t y0, uint32_t y1) {
    CK(cudaSetDevice(device_));
    if (!d_image_ || !W_ || !H_) throw CudaError{ B200PT_ERR_NO_SCENE, "PostProcess without an input image" };
    post_chain(d_image_.get(), y0, y1);
    post_denoised_ = false;
}
void Engine::post_chain(const float4 *src, uint32_t y0, uint32_t y1) {
    if (world_ != 1) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "post_process needs the full image: gather the bands first (world must be 1)" };
    if (y0 >= y1 || y1 > H_) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "post_process_rows: bad row range" };
    ensure_post();
    join_waves();
    const bool whole = (y0 == 0 && y1 == H_);
    const uint32_t levels = (uint32_t)d_mips_.size();
    const uint32_t mips = std::min(std::max(bloom_.MipCount, 1u), levels);                      // :195
    const PostParams p{ tonemap_.Exposure, tonemap_.Gamma, bloom_.BloomThreshold, bloom_.BloomStrength, bloom_.FalloffRange };
    // Fused chain (default): mip 0 is never materialised -- the threshold is evaluated inside the first down pass and inside the final
    // [up + tonemap] kernel.  B200PT_POST_FUSED=0 (or a 1-level chain) runs the reference's pass-per-pass structure; both produce the
    // same RGBA8 image bit for bit (tested).
    bool fused = mips >= 2;
    if (const char *e = getenv("B200PT_POST_FUSED")) { if (atoi(e) == 0) fused = false; }
    if (!fused && !whole) throw CudaError{ B200PT_ERR_NOT_IMPLEMENTED, "post_process_rows needs the fused chain (MipCount >= 2, B200PT_POST_FUSED unset)" };
    if (fused) {
        // needed row ranges, inclusive: U[i] post-up rows of mip i, D[i] down-result rows of mip i (i = 1 .. mips-1)
        int U[24][2], D[24][2];
        auto hgt = [&](uint32_t i) { return (int)mip_wh_[2 * i + 1]; };
        auto clampr = [&](int v, uint32_t i) { return std::min(std::max(v, 0), hgt(i) - 1); };
        {   // mip 0 rows the final kernel builds for outputs [y0, y1): y-1 .. y (bilinear bloom fetch); their up-sample term reads mip 1 rows yy/2 - 1 .. yy/2 + 2
            const int a = std::max((int)y0 - 1, 0), b = (int)y1 - 1;
            U[1][0] = clampr(a / 2 - 1, 1); U[1][1] = clampr(b / 2 + 2, 1);
        }
        for (uint32_t i = 2; i < mips; i++) { U[i][0] = clampr(U[i - 1][0] / 2 - 1, i); U[i][1] = clampr(U[i - 1][1] / 2 + 2, i); }   // up pass i: dst rows U[i-1] read src rows y/2 - 1 .. y/2 + 2
        D[mips - 1][0] = U[mips - 1][0]; D[mips - 1][1] = U[mips - 1][1];
        for (uint32_t i = mips - 1; i-- > 1;) {                                                 // down pass i+1: dst rows D[i+1] read src rows 2y - 2 .. 2y + 1
            D[i][0] = std::min(U[i][0], clampr(2 * D[i + 1][0] - 2, i)); D[i][1] = std::max(U[i][1], clampr(2 * D[i + 1][1] + 1, i));
        }
        auto rows_of = [&](const int r[2], int out[2]) { out[0] = r[0]; out[1] = r[1] + 1; };
        int r[2];
        rows_of(D[1], r);
        launch_bloom_down_first(src, W_, H_, d_mips_[1].get(), mip_wh_[2], mip_wh_[3], p, stream_, whole ? nullptr : r);                               // :200-226, i == 0 and i == 1
        for (uint32_t i = 2; i < mips; i++) { rows_of(D[i], r); launch_bloom_down(d_mips_[i - 1].get(), mip_wh_[2 * (i - 1)], mip_wh_[2 * (i - 1) + 1], d_mips_[i].get(), mip_wh_[2 * i], mip_wh_[2 * i + 1], p, stream_, whole ? nullptr : r); }
        for (uint32_t i = mips - 1; i > 1; i--) { rows_of(U[i - 1], r); launch_bloom_up(d_mips_[i].get(), mip_wh_[2 * i], mip_wh_[2 * i + 1], d_mips_[i - 1].get(), mip_wh_[2 * (i - 1)], mip_wh_[2 * (i - 1) + 1], p, stream_, whole ? nullptr : r); }   // :229-235
        r[0] = (int)y0; r[1] = (int)y1;
        launch_bloom_final(src, d_mips_[1].get(), mip_wh_[2], mip_wh_[3], d_ldr_.get(), (keep_bloom_ && whole) ? d_mips_[0].get() : nullptr, W_, H_, p, stream_, whole ? nullptr : r);   // last up pass + :238-245
        bloom_valid_ = keep_bloom_ && whole;
    } else {
        launch_bloom_threshold(src, d_mips_[0].get(), W_ * H_, p, tree_.lc.grid_light > 0 ? tree_.lc.grid_light : 1184, stream_);            // :200-226, i == 0
        for (uint32_t i = 1; i < mips; i++) launch_bloom_down(d_mips_[i - 1].get(), mip_wh_[2 * (i - 1)], mip_wh_[2 * (i - 1) + 1], d_mips_[i].get(), mip_wh_[2 * i], mip_wh_[2 * i + 1], p, stream_);
        for (uint32_t i = mips - 1; i > 0; i--) launch_bloom_up(d_mips_[i].get(), mip_wh_[2 * i], mip_wh_[2 * i + 1], d_mips_[i - 1].get(), mip_wh_[2 * (i - 1)], mip_wh_[2 * (i - 1) + 1], p, stream_);   // :229-235
        launch_tonemap(src, d_mips_[0].get(), d_ldr_.get(), W_, H_, p, stream_);                           // :238-245
        bloom_valid_ = true;
    }
    CK(cudaGetLastError());
}
void Engine::get_ldr_rows(uint32_t y0, uint32_t y1, uint8_t *dst, bool dev) {
    CK(cudaSetDevice(device_));
    if (!d_ldr_ || !dst || y0 >= y1 || y1 > H_) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "post_process has not run / bad row range" };
    CK(cudaMemcpyAsync(dst, reinterpret_cast<const uint8_t *>(d_ldr_.get()) + (size_t)y0 * W_ * 4, (size_t)(y1 - y0) * W_ * 4, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream_));
    if (!dev) CK(cudaStreamSynchronize(stream_));
}
void Engine::get_ldr(uint8_t *dst, bool dev) {
    CK(cudaSetDevice(device_));
    if (!d_ldr_ || !dst) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "post_process has not run" };
    CK(cudaMemcpyAsync(dst, d_ldr_.get(), (size_t)W_ * H_ * 4, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
}
void Engine::get_bloom(float *dst) {
    CK(cudaSetDevice(device_));
    if (d_mips_.empty() || !dst) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "post_process has not run" };
    if (!bloom_valid_) {                                                     // the fused chain skips mip 0 until somebody asks for it: re-run it on the same input
        keep_bloom_ = true;
        if (post_denoised_ && has_denoised()) post_chain(d_dn_.get() + 2 * dn_pixels_, 0, H_); else post_process();
    }
    CK(cudaMemcpyAsync(dst, d_mips_[0].get(), (size_t)W_ * H_ * sizeof(float4), cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
}

void Engine::volume_walks(uint32_t n, const float *org, const float *dir, const uint32_t *seeds, float ray_depth, float *T, float *scatter, int32_t *vol, uint32_t *rng2) {
    CK(cudaSetDevice(device_));
    if (!n) return;
    sync_all();
    DeviceBlocks a(stream_);
    float *d_T = a.out<float>(n), *d_s = a.out<float>(n); int32_t *d_v = a.out<int32_t>(n); uint32_t *d_r = a.out<uint32_t>(2 * (size_t)n);
    launch_volume_walks(dev_scene(), n, a.in(org, 3 * (size_t)n), a.in(dir, 3 * (size_t)n), a.in(seeds, n), ray_depth, d_T, d_s, d_v, d_r, stream_);
    a.get(T, d_T, n); a.get(scatter, d_s, n); a.get(vol, d_v, n); a.get(rng2, d_r, 2 * (size_t)n);
    a.sync();
}
// The closest-hit walk of trace_query in the shape the render's one-ray-per-thread kernels take for this scene, with one [tmin, tmax] for all rays.
// stats: nodes visited and triangles tested per ray.
void Engine::trace_closest(uint32_t n, const float *org, const float *dir, float tmin, float tmax, float *t, uint32_t *prim, uint32_t *inst, float *uv, uint32_t *stats) {
    const std::vector<float> lo(n, tmin), hi(n, tmax);
    std::vector<uint32_t> st3(stats ? 3 * (size_t)n : 0);
    const int shape = tree_.lc.bvh_in_smem ? (tree_.n_flat ? TQ_FLAT : TQ_SHARED) : TQ_GLOBAL;
    trace_query(shape, TQ_CLOSEST, false, n, org, dir, lo.data(), hi.data(), nullptr, nullptr, t, prim, inst, uv, nullptr, stats ? st3.data() : nullptr);
    if (stats) for (size_t i = 0; i < n; i++) { stats[2 * i] = st3[3 * i]; stats[2 * i + 1] = st3[3 * i + 1]; }
}
void Engine::trace_query(int shape, int kind, bool fma, uint32_t n, const float *org, const float *dir, const float *tmin, const float *tmax, const uint32_t *target,
                         const float *tmax_test, float *t, uint32_t *prim, uint32_t *inst, float *uv, uint32_t *occluded, uint32_t *stats) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!n) return;
    DeviceBlocks a(stream_);
    const bool any = kind != TQ_CLOSEST, tgt = kind == TQ_TARGET;
    TraceQuery q{};
    q.n = n;
    q.org = a.in(org, 3 * (size_t)n); q.dir = a.in(dir, 3 * (size_t)n); q.tmin = a.in(tmin, n); q.tmax = a.in(tmax, n);
    if (tgt) { q.target = a.in(target, n); q.tmax_test = a.in(tmax_test, n); }
    if (any) q.occluded = a.out<uint32_t>(n);
    else { q.t = a.out<float>(n); q.prim = a.out<uint32_t>(n); q.inst = a.out<uint32_t>(n); q.uv = a.out<float>(2 * (size_t)n); }
    if (stats) q.stats = a.out<uint32_t>(3 * (size_t)n);
    const int r = launch_trace_query(tree_.lc, dev_scene(), tree_.bvh.depth4, shape, kind, fma, q, stream_);
    if (r == TQ_UNSUPPORTED) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "trace_query: the scene has no such traversal shape" };
    CK((cudaError_t)r);
    if (any) a.get(occluded, q.occluded, n);
    else { a.get(t, q.t, n); a.get(prim, q.prim, n); a.get(inst, q.inst, n); a.get(uv, q.uv, 2 * (size_t)n); }
    if (stats) a.get(stats, q.stats, 3 * (size_t)n);
    a.sync();
}
void Engine::shade_query(bool force_general, uint32_t n, const uint32_t *inst, const uint32_t *prim, const float *uv, const float *dir, const float *org,
                         const float *pay_pdf, const uint32_t *rng, const float *L, float *out) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!has_env() || !has_luts()) throw CudaError{ B200PT_ERR_NO_SCENE, "shade_query: no environment map or no lookup tables" };
    if (!n) return;
    const DevScene sc = dev_scene();
    if (sc.n_volumes != 0u || atmosphere_.Enable) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "shade_query: scenes with volumes or the atmosphere are not supported" };
    std::vector<uint32_t> gid(n);
    for (uint32_t i = 0; i < n; i++) {                                      // (instance, primitive) -> global triangle id, as k_world_tris numbers them
        if (inst[i] >= h_instances_.size() || prim[i] >= h_meshes_[h_instances_[inst[i]].mesh].tri_count)
            throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "shade_query: instance or primitive out of range" };
        gid[i] = h_instances_[inst[i]].tri_base + prim[i];
    }
    DeviceBlocks a(stream_);
    ShadeQuery q{};
    q.n = n; q.force_general = force_general;
    q.gid = a.in(gid.data(), n); q.rng = a.in(rng, n);
    q.uv = a.in(uv, 2 * (size_t)n); q.dir = a.in(dir, 3 * (size_t)n); q.org = a.in(org, 3 * (size_t)n);
    q.pay_pdf = a.in(pay_pdf, n);
    if (L) q.L = a.in(L, 3 * (size_t)n);
    const size_t out_count = (size_t)n * B200PT_SQ_STRIDE;
    q.out = a.out<float>(out_count);
    CK((cudaError_t)launch_shade_query(sc, make_dev_config(), q, stream_));
    a.get(out, q.out, out_count);
    a.sync();
}
void Engine::miss_query(uint32_t n, const float *dir, const uint32_t *depth, const float *pay_pdf, float *out) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!has_env()) throw CudaError{ B200PT_ERR_NO_SCENE, "miss_query: no environment map" };
    if (!n) return;
    DeviceBlocks a(stream_);
    MissQuery q{};
    q.n = n;
    q.dir = a.in(dir, 3 * (size_t)n); q.depth = a.in(depth, n); q.pay_pdf = a.in(pay_pdf, n);
    const size_t out_count = (size_t)n * B200PT_MQ_STRIDE;
    q.out = a.out<float>(out_count);
    CK((cudaError_t)launch_miss_query(dev_scene(), make_dev_config(), q, stream_));
    a.get(out, q.out, out_count);
    a.sync();
}
void Engine::bounce_query(uint32_t n, const float *in, uint32_t flags, float *out, uint32_t *survivors) {
    CK(cudaSetDevice(device_));
    if (!has_scene_) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!has_env() || !has_luts()) throw CudaError{ B200PT_ERR_NO_SCENE, "bounce_query: no environment map or no lookup tables" };
    DevScene sc = dev_scene();
    if (sc.n_volumes != 0u || atmosphere_.Enable) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bounce_query: scenes with volumes or the atmosphere are not supported" };
    static_assert(B200PT_BQ_STORE == WAVE_STORE && B200PT_BQ_CARRY == WAVE_CARRY, "bounce_query flags are the wave flags");
    if (flags & ~(uint32_t)(B200PT_BQ_STORE | B200PT_BQ_CARRY)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bounce_query: unknown flag bits" };
    *survivors = 0;
    if (!n) return;
    constexpr uint32_t IN = B200PT_BQ_IN_STRIDE, OUT = B200PT_BQ_OUT_STRIDE;
    std::vector<float4> org_pdf(n), dir_rng(n), thr_depth(n), rad_slot(n), medium(n), sample(n);
    std::vector<float> medium_g(n);
    for (uint32_t i = 0; i < n; i++) {
        const float *r = in + (size_t)i * IN;
        const float *o = r + B200PT_BQ_IN_ORG, *d = r + B200PT_BQ_IN_DIR;
        uint32_t dflags; memcpy(&dflags, r + B200PT_BQ_IN_DFLAGS, 4);
        if (!std::isfinite(o[0]) || !std::isfinite(o[1]) || !std::isfinite(o[2])) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bounce_query: non-finite origin" };
        if (!std::isfinite(d[0]) || !std::isfinite(d[1]) || !std::isfinite(d[2]) || (d[0] == 0.0f && d[1] == 0.0f && d[2] == 0.0f))
            throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bounce_query: zero or non-finite direction" };
        if ((dflags & 0x07FFFFFFu) >= cfg_.MaxDepth) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bounce_query: Depth >= MaxDepth" };
        if (dflags & (3u << 29)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bounce_query: DFLAGS bits 29-30 set" };
        org_pdf[i] = make_float4(o[0], o[1], o[2], r[B200PT_BQ_IN_PDF]);
        dir_rng[i] = make_float4(d[0], d[1], d[2], r[B200PT_BQ_IN_RNG]);
        thr_depth[i] = make_float4(r[B200PT_BQ_IN_THR], r[B200PT_BQ_IN_THR + 1], r[B200PT_BQ_IN_THR + 2], r[B200PT_BQ_IN_DFLAGS]);
        float slot; memcpy(&slot, &i, 4);
        rad_slot[i] = make_float4(r[B200PT_BQ_IN_RAD], r[B200PT_BQ_IN_RAD + 1], r[B200PT_BQ_IN_RAD + 2], slot);
        memcpy(&medium[i], r + B200PT_BQ_IN_MEDIUM, 16); medium_g[i] = r[B200PT_BQ_IN_MEDIUM_G];
        memcpy(&sample[i], r + B200PT_BQ_IN_SAMPLE, 16);
    }
    sync_all();                                               // the wave buffers of context 0 may still serve a wave in flight
    ensure_wave(n, 1);
    WaveBuf &B = wb_[0];
    const PathState pst[2] = { { B.ps[0].org_pdf, B.ps[0].dir_rng, B.ps[0].thr_depth, B.ps[0].rad_slot, B.ps[0].medium, B.ps[0].medium_g, nullptr },
                               { B.ps[1].org_pdf, B.ps[1].dir_rng, B.ps[1].thr_depth, B.ps[1].rad_slot, B.ps[1].medium, B.ps[1].medium_g, nullptr } };
    const int cur = 1; const uint32_t k = 1;                  // a non-primary bounce: control word k & 1 holds the live count
    const size_t b4 = (size_t)n * sizeof(float4);
    CK(cudaMemcpyAsync(pst[cur].org_pdf, org_pdf.data(), b4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(pst[cur].dir_rng, dir_rng.data(), b4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(pst[cur].thr_depth, thr_depth.data(), b4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(pst[cur].rad_slot, rad_slot.data(), b4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(pst[cur].medium, medium.data(), b4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(pst[cur].medium_g, medium_g.data(), (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(B.sample_buf, sample.data(), b4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemsetAsync(B.rng_carry, 0, (size_t)n * 4, stream_));
    CK(cudaMemsetAsync(B.counts.get(), 0, CTRL_WORDS * sizeof(uint32_t), stream_));
    CK(cudaMemcpyAsync(B.counts.get() + (k & 1u), &n, 4, cudaMemcpyHostToDevice, stream_));
    CK(cudaStreamSynchronize(stream_));                       // (the pageable sources above are copied by now)

    const DevConfig dc = make_dev_config();
    const CallPlan cp = plan_call(tree_.lc, sc, dc, scene_has_media(), class_mask_);
    sc.pre_pass = 0u;
    last_.kernel_launches += bounce(cp, sc, dc, B, pst, cur, k, flags, stream_, [](int) {});

    std::vector<float4> hit(n), nx_op(n), nx_dr(n), nx_td(n), nx_rs(n), nx_med(n);
    std::vector<float> nx_g(n);
    std::vector<uint32_t> carry(n), ctrl(CTRL_WORDS);
    const PathState &dst = pst[cur ^ 1];
    CK(cudaMemcpyAsync(ctrl.data(), B.counts.get(), CTRL_WORDS * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(hit.data(), B.so.hit, b4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(sample.data(), B.sample_buf, b4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(carry.data(), B.rng_carry, (size_t)n * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    const uint32_t m = ctrl[(k & 1u) ^ 1u];
    *survivors = m;
    if (m > n) throw CudaError{ B200PT_ERR_CUDA, "bounce_query: more survivors than paths" };
    if (m) {
        const size_t m4 = (size_t)m * sizeof(float4);
        CK(cudaMemcpyAsync(nx_op.data(), dst.org_pdf, m4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaMemcpyAsync(nx_dr.data(), dst.dir_rng, m4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaMemcpyAsync(nx_td.data(), dst.thr_depth, m4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaMemcpyAsync(nx_rs.data(), dst.rad_slot, m4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaMemcpyAsync(nx_med.data(), dst.medium, m4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaMemcpyAsync(nx_g.data(), dst.medium_g, (size_t)m * 4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));
    }
    CK(cudaGetLastError());
    memset(out, 0, (size_t)n * OUT * sizeof(float));
    for (uint32_t i = 0; i < n; i++) {
        float *r = out + (size_t)i * OUT;
        uint32_t gid; memcpy(&gid, &hit[i].w, 4);
        uint32_t inst = 0xFFFFFFFFu, prim = 0xFFFFFFFFu;
        if (gid < n_tris_) {                                  // instance-major triangle id -> (instance, primitive of its mesh)
            const auto it = std::upper_bound(h_instances_.begin(), h_instances_.end(), gid, [](uint32_t g, const DevInstance &a) { return g < a.tri_base; });
            inst = (uint32_t)(it - h_instances_.begin()) - 1u; prim = gid - h_instances_[inst].tri_base;
        }
        r[B200PT_BQ_OUT_T] = hit[i].x; r[B200PT_BQ_OUT_U] = hit[i].y; r[B200PT_BQ_OUT_V] = hit[i].z;
        memcpy(r + B200PT_BQ_OUT_INST, &inst, 4); memcpy(r + B200PT_BQ_OUT_PRIM, &prim, 4);
        memcpy(r + B200PT_BQ_OUT_SAMPLE, &sample[i], 16); memcpy(r + B200PT_BQ_OUT_CARRY, &carry[i], 4);
    }
    for (uint32_t j = 0; j < m; j++) {                        // the survivors in compacted order, each to the record of its slot
        uint32_t slot; memcpy(&slot, &nx_rs[j].w, 4);
        if (slot >= n) throw CudaError{ B200PT_ERR_CUDA, "bounce_query: a survivor carries a slot out of range" };
        float *r = out + (size_t)slot * OUT, *s = r + B200PT_BQ_OUT_NEXT;
        r[B200PT_BQ_OUT_ALIVE] += 1.0f;                       // (a slot written twice reads 2)
        memcpy(s + B200PT_BQ_IN_ORG, &nx_op[j], 16); memcpy(s + B200PT_BQ_IN_DIR, &nx_dr[j], 16);
        memcpy(s + B200PT_BQ_IN_THR, &nx_td[j], 16); memcpy(s + B200PT_BQ_IN_RAD, &nx_rs[j], 16);
        uint32_t df; memcpy(&df, &nx_td[j].w, 4);
        if (df >> 31) { memcpy(s + B200PT_BQ_IN_MEDIUM, &nx_med[j], 16); s[B200PT_BQ_IN_MEDIUM_G] = nx_g[j]; }
    }
}
// LookupTableCalculator::CalculateTable (PT/LookupTableCalculator.cpp:44-157) on this engine's device and stream.
// slices == 0 picks enough dispatch slices to give every SM ~2048 resident threads.
void Engine::bake_lut(int kind, uint32_t sx, uint32_t sy, uint32_t sz, uint32_t sample_count, uint32_t seed, uint32_t slices, float *out_host, float *elapsed_ms) {
    CK(cudaSetDevice(device_));
    if (kind < 0 || kind > 2 || !sx || !sy || !sz || !out_host || (uint64_t)sx * sy * sz > (1ull << 28)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bake_lut: bad arguments" };
    const size_t n = (size_t)sx * sy * sz;
    if (!slices) {
        cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, device_));
        const size_t want = (size_t)prop.multiProcessorCount * 2048;
        slices = (uint32_t)std::max<size_t>(1, (want + n - 1) / n);
    }
    slices = std::min<uint32_t>(slices, 4096u);
    DevPtr<float> d_part, d_tab;
    CK(alloc(d_part, n * slices * sizeof(float)));
    if (alloc(d_tab, n * sizeof(float)) != cudaSuccess) throw CudaError{ B200PT_ERR_OUT_OF_MEMORY, "bake_lut: out of device memory" };
    const Event e0 = make_event(cudaEventDefault), e1 = make_event(cudaEventDefault);
    CK(cudaEventRecord(e0.get(), stream_));
    launch_bake_lut(kind, d_part.get(), d_tab.get(), sx, sy, sz, sample_count, seed, slices, stream_);
    CK(cudaEventRecord(e1.get(), stream_));
    CK(cudaMemcpyAsync(out_host, d_tab.get(), n * sizeof(float), cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    float ms = 0.0f; CK(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
    if (elapsed_ms) *elapsed_ms = ms;
}
// ---------------------------------------------------------------- denoiser (denoise_kernels.cu, DESIGN.md section 12)
static void check_denoise_params(const b200pt_denoise_params &p) {
    if (p.Iterations > 10) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "denoise Iterations must be <= 10" };
    if (p.FeatureSamples == 0 || p.FeatureSamples > 256) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "denoise FeatureSamples must be 1 .. 256" };
    for (float v : { p.SigmaLuminance, p.SigmaNormal, p.SigmaDepth })
        if (!std::isfinite(v) || v < 0.0f) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "denoise sigmas must be finite and >= 0" };
}
static uint32_t pcg_host(uint32_t in) { const uint32_t st = in * 747796405u + 2891336453u; const uint32_t w = ((st >> ((st >> 28u) + 4u)) ^ st) * 277803737u; return (w >> 22u) ^ w; }
void Engine::free_denoise() { d_dn_.reset(); dn_pixels_ = 0; dn_w_ = dn_h_ = 0; }   // (d_dn_img_ is sized by the caller's images: freed with the engine)
void Engine::ensure_denoise() {
    const size_t n = (size_t)W_ * local_rows_;
    if (d_dn_ && n == dn_pixels_) return;
    sync_all();
    free_denoise();
    CK(alloc(d_dn_, std::max<size_t>(n, 1) * (6 * sizeof(float4) + sizeof(float))));
    dn_pixels_ = n;
}
void Engine::run_features(const b200pt_denoise_params &p) {
    if (!has_scene_ || !d_image_) throw CudaError{ B200PT_ERR_NO_SCENE, "denoise needs a scene and an image" };
    if (!records()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "denoise needs per-pixel statistics (b200pt_set_track_variance) or adaptive sampling" };
    ensure_denoise();
    prepare_adaptive();
    join_waves();
    const size_t n = dn_pixels_;
    if (!n) return;
    // forward: the view direction of the image centre (camera_ray with dx = dy = 0, no jitter), the axis of the view depth
    const float *PI = proj_inv_, *VI = view_inv_;
    double t[3] = { (double)PI[8] + PI[12], (double)PI[9] + PI[13], (double)PI[10] + PI[14] }, d[3];
    const double tl = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    for (int k = 0; k < 3; k++) d[k] = (VI[k] * t[0] + VI[4 + k] * t[1] + VI[8 + k] * t[2]) / tl;
    const double dl = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    const float3 fwd = make_float3((float)(d[0] / dl), (float)(d[1] / dl), (float)(d[2] / dl));
    CK((cudaError_t)launch_features(tree_.lc, dev_scene(), make_dev_config(), fwd, p.FeatureSamples, pcg_host(0x46454154u), d_dn_.get(), d_dn_.get() + n, stream_));
    launch_record_variance(d_px_state_.get(), (uint32_t)n, reinterpret_cast<float *>(d_dn_.get() + 6 * n), stream_);
    CK(cudaGetLastError());
}
void Engine::denoise(const b200pt_denoise_params &p, float *elapsed_ms) {
    CK(cudaSetDevice(device_));
    check_denoise_params(p);
    if (world_ != 1) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "denoise needs the full image (world 1): gather b200pt_get_denoise_inputs and use b200pt_denoise_image" };
    const Event e0 = make_event(cudaEventDefault), e1 = make_event(cudaEventDefault);
    join_waves();                                             // the timed window starts behind the render's waves
    CK(cudaEventRecord(e0.get(), stream_));
    run_features(p);
    const size_t n = dn_pixels_;
    launch_denoise_filter(W_, H_, d_image_.get(), d_dn_.get(), d_dn_.get() + n, reinterpret_cast<const float *>(d_dn_.get() + 6 * n), p.Iterations, p.SigmaLuminance, p.SigmaNormal,
                          p.SigmaDepth, d_dn_.get() + 3 * n, d_dn_.get() + 2 * n, stream_);
    CK(cudaEventRecord(e1.get(), stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    float ms = 0.0f; CK(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
    if (elapsed_ms) *elapsed_ms = ms;
    dn_w_ = W_; dn_h_ = H_;
}
void Engine::get_denoised(float *dst, bool dev) {
    CK(cudaSetDevice(device_));
    if (!dst || !has_denoised()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "no denoised image of the current size (b200pt_denoise first)" };
    CK(cudaMemcpyAsync(dst, d_dn_.get() + 2 * dn_pixels_, (size_t)W_ * H_ * sizeof(float4), dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
}
void Engine::denoise_inputs(const b200pt_denoise_params &p, float *albedo_cov, float *normal_depth, float *variance) {
    CK(cudaSetDevice(device_));
    check_denoise_params(p);
    run_features(p);
    const size_t n = dn_pixels_;
    if (albedo_cov) CK(cudaMemcpyAsync(albedo_cov, d_dn_.get(), n * sizeof(float4), cudaMemcpyDeviceToHost, stream_));
    if (normal_depth) CK(cudaMemcpyAsync(normal_depth, d_dn_.get() + n, n * sizeof(float4), cudaMemcpyDeviceToHost, stream_));
    if (variance) CK(cudaMemcpyAsync(variance, d_dn_.get() + 6 * n, n * sizeof(float), cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
}
void Engine::denoise_image(uint32_t w, uint32_t h, const float *color, const float *albedo_cov, const float *normal_depth, const float *variance,
                           const b200pt_denoise_params &p, float *out, bool dev) {
    CK(cudaSetDevice(device_));
    check_denoise_params(p);
    if (!w || !h || w > 65535 || h > 65535) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "bad image size" };
    const size_t n = (size_t)w * h, bytes = n * (dev ? 3 : 7) * sizeof(float4) + (dev ? 0 : n * sizeof(float));
    if (bytes > dn_img_bytes_) {                              // kept for the next call: repeated calls allocate nothing
        sync_all(); dn_img_bytes_ = 0;
        CK(alloc(d_dn_img_, bytes)); dn_img_bytes_ = bytes;
    }
    float4 *const buf = d_dn_img_.get();                            // [scratch 3n | device copies of the inputs and the output when they are host memory]
    const float4 *c = reinterpret_cast<const float4 *>(color), *a = reinterpret_cast<const float4 *>(albedo_cov), *nd = reinterpret_cast<const float4 *>(normal_depth);
    const float *v = variance; float4 *o = reinterpret_cast<float4 *>(out);
    cudaError_t e = cudaSuccess;
    if (!dev) {
        float4 *hc = buf + 3 * n, *ha = buf + 4 * n, *hn = buf + 5 * n; float *hv = reinterpret_cast<float *>(buf + 7 * n);
        if (e == cudaSuccess) e = cudaMemcpyAsync(hc, color, n * sizeof(float4), cudaMemcpyHostToDevice, stream_);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ha, albedo_cov, n * sizeof(float4), cudaMemcpyHostToDevice, stream_);
        if (e == cudaSuccess) e = cudaMemcpyAsync(hn, normal_depth, n * sizeof(float4), cudaMemcpyHostToDevice, stream_);
        if (e == cudaSuccess) e = cudaMemcpyAsync(hv, variance, n * sizeof(float), cudaMemcpyHostToDevice, stream_);
        c = hc; a = ha; nd = hn; v = hv; o = buf + 6 * n;
    }
    if (e == cudaSuccess) {
        launch_denoise_filter(w, h, c, a, nd, v, p.Iterations, p.SigmaLuminance, p.SigmaNormal, p.SigmaDepth, buf, o, stream_);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && !dev) e = cudaMemcpyAsync(out, o, n * sizeof(float4), cudaMemcpyDeviceToHost, stream_);
    const cudaError_t es = cudaStreamSynchronize(stream_);
    CK(e); CK(es);
}
void Engine::post_process_denoised() {
    CK(cudaSetDevice(device_));
    if (!has_denoised()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "no denoised image of the current size (b200pt_denoise first)" };
    post_chain(d_dn_.get() + 2 * dn_pixels_, 0, H_);
    post_denoised_ = true;
}
void Engine::scene_stats(uint32_t *tris, uint32_t *nodes, uint32_t *emissive, uint32_t *textures) const {
    if (tris) *tris = n_tris_; if (nodes) *nodes = tree_.bvh.n_nodes; if (emissive) *emissive = n_emissive_; if (textures) *textures = (uint32_t)scene_.textures.size();
}

// The launchers update_instance_transforms(B200PT_REBUILD_GPU) runs, on the caller's boxes in the given order (no scene needed).  Rejects what
// bvh2_ploc_build_host rejects: nothing is written but zero counts.
void Engine::ploc_build_query(const float *ref_boxes, uint32_t n, BvhNode *nodes_out, uint32_t *perm_out, uint32_t *n_out, int *depth_out,
                              Bvh4Node *nodes4_out, uint32_t *n4_out, int *depth4_out) {
    CK(cudaSetDevice(device_));
    *n_out = 0; *depth_out = 0; *n4_out = 0; *depth4_out = 0;
    for (size_t i = 0; i < (size_t)n; i++)
        for (int a = 0; a < 3; a++) if (!(ref_boxes[i * 6 + a] <= ref_boxes[i * 6 + 3 + a])) return;
    DeviceBlocks a(stream_);
    const float *box = a.in(ref_boxes, (size_t)n * 6);
    BvhNode *nodes = a.out<BvhNode>(n - 1); uint32_t *perm = a.out<uint32_t>(n);
    uint32_t n2 = 0; int d2 = 0;
    int r = ploc_build(box, n, nodes, perm, &n2, &d2, h_small_.get(), stream_);
    if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("ploc_build failed: ") + cudaGetErrorString((cudaError_t)r) };
    if (n2 == 0) return;
    Bvh4Node *nodes4 = a.out<Bvh4Node>(n2);
    uint32_t n4 = 0; int d4 = 0;
    r = bvh4_collapse_device(nodes, n2, 0, nodes4, &n4, &d4, h_small_.get(), stream_);
    if (r != 0) throw CudaError{ B200PT_ERR_CUDA, std::string("bvh4_collapse_device failed: ") + cudaGetErrorString((cudaError_t)r) };
    a.get(nodes_out, nodes, n2); a.get(perm_out, perm, n);
    if (n4) a.get(nodes4_out, nodes4, n4);
    a.sync();
    *n_out = n2; *depth_out = d2; *n4_out = n4; *depth4_out = d4;
}

} // namespace b200pt
