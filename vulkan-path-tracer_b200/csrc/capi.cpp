// capi.cpp -- the extern "C" boundary declared in include/b200pt.h.
// Error behaviour mirrors VulkanHelper's Expected<T, VHResult> (VulkanHelper/Include/Core/Error.h:14-72): every entry
// point returns a code, nothing aborts (the reference's VH_ASSERT -> std::terminate, Log.h:118-123, is NOT reproduced),
// and no exception crosses the boundary.
#include "engine.h"
#include <cstring>
#include <cstdlib>
#include <new>
#include <cmath>
#include <functional>

using namespace b200pt;

struct b200pt_s { Engine *eng = nullptr; std::string err; };

static thread_local std::string g_err;

template <class F> static int32_t guard(b200pt_handle h, F &&f) {
    if (!h || !h->eng) return B200PT_ERR_WRONG_ARGUMENTS;
    try { f(*h->eng); return B200PT_OK; }
    catch (const CudaError &e) { h->err = e.what; return e.code < 0 ? e.code : B200PT_ERR_CUDA; }
    catch (const std::bad_alloc &) { h->err = "host out of memory"; return B200PT_ERR_OUT_OF_MEMORY; }
    catch (const std::exception &e) { h->err = e.what(); return B200PT_ERR_UNKNOWN; }
    catch (...) { h->err = "unknown error"; return B200PT_ERR_UNKNOWN; }
}

static_assert(sizeof(b200pt_volume) == 148 && sizeof(b200pt_density_grid) == 80, "b200pt_volume / b200pt_density_grid layout (binding.py, INTEGRATION.md)");
static_assert(sizeof(b200pt_adaptive) == 16, "b200pt_adaptive layout (binding.py, checkpoint version 2)");
static_assert(sizeof(b200pt_denoise_params) == 20, "b200pt_denoise_params layout (binding.py)");

extern "C" {

const char *b200pt_version(void) { return "b200pt 0.1 (sm_90a wavefront path tracer)"; }

int32_t b200pt_create(int32_t device, b200pt_handle *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    *out = nullptr;
    b200pt_s *h = new (std::nothrow) b200pt_s();
    if (!h) return B200PT_ERR_OUT_OF_MEMORY;
    try { h->eng = new Engine(device); }
    catch (const CudaError &e) { g_err = e.what; int c = e.code < 0 ? e.code : B200PT_ERR_CUDA; delete h; return c; }
    catch (...) { delete h; return B200PT_ERR_UNKNOWN; }
    *out = h;
    return B200PT_OK;
}
int32_t b200pt_destroy(b200pt_handle h) { if (!h) return B200PT_ERR_WRONG_ARGUMENTS; try { delete h->eng; } catch (...) {} delete h; return B200PT_OK; }
const char *b200pt_last_error(b200pt_handle h) { return h ? h->err.c_str() : g_err.c_str(); }

int32_t b200pt_set_scene_file(b200pt_handle h, const char *path) {
    if (!path) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        HostScene sc; std::string err;
        if (!load_scene_file(path, sc, err)) throw CudaError{ B200PT_ERR_INIT_FAILED, "Failed to import scene: " + err };
        e.set_scene(std::move(sc));
    });
}
int32_t b200pt_set_scene_arrays(b200pt_handle h, const b200pt_scene_desc *d) {
    return guard(h, [&](Engine &e) {
        HostScene sc; std::string err;
        if (!scene_from_desc(d, sc, err)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, err };
        e.set_scene(std::move(sc));
    });
}
int32_t b200pt_set_env_map_file(b200pt_handle h, const char *path) {
    if (!path) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        std::vector<float> px; uint32_t w, hh; std::string err;
        if (!decode_hdr_rgba32f(path, w, hh, px, err)) throw CudaError{ B200PT_ERR_INIT_FAILED, err };
        e.set_env_map(w, hh, px.data());
    });
}
int32_t b200pt_set_env_map(b200pt_handle h, uint32_t w, uint32_t hh, const float *rgba) { return guard(h, [&](Engine &e) { e.set_env_map(w, hh, rgba); }); }
int32_t b200pt_set_luts(b200pt_handle h, const float *a, const float *b, const float *c) { return guard(h, [&](Engine &e) { e.set_luts(a, b, c); }); }
int32_t b200pt_set_luts_dir(b200pt_handle h, const char *dir) {
    if (!dir) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        const char *names[3] = { "ReflectionLookup.bin", "RefractionLookupHitFromOutside.bin", "RefractionLookupHitFromInside.bin" };   // PathTracer.cpp:199-201
        const size_t n[3] = { 64 * 64 * 32, 128 * 128 * 32, 128 * 128 * 32 };
        std::vector<float> t[3];
        for (int i = 0; i < 3; i++) {
            std::string p = std::string(dir) + "/" + names[i];
            FILE *f = fopen(p.c_str(), "rb");
            if (!f) throw CudaError{ B200PT_ERR_INIT_FAILED, "Failed to open lookup table " + p };
            t[i].resize(n[i]); size_t got = fread(t[i].data(), 4, n[i], f); fclose(f);
            if (got != n[i]) throw CudaError{ B200PT_ERR_INIT_FAILED, "short lookup table " + p };
        }
        e.set_luts(t[0].data(), t[1].data(), t[2].data());
    });
}

int32_t b200pt_default_config(b200pt_config *c) {
    if (!c) return B200PT_ERR_WRONG_ARGUMENTS;
    memset(c, 0, sizeof *c);                                        // PathTracer.h:197-233
    c->SamplesPerFrame = 1; c->MaxDepth = 200; c->MaxLuminance = 500.0f; c->FocusDistance = 1.0f; c->DepthOfFieldStrength = 0.0f;
    c->SkyRotationAzimuth = 0.0f; c->SkyRotationAltitude = 0.0f; c->SkyIntensity = 1.0f; c->EmissiveMeshSamplingPDFBias = 0.0f;
    c->ScreenChunkCount = 1; c->EnableSkyMIS = 1; c->EnableMeshMIS = 1; c->ShowEnvMapDirectly = 1; c->UseOnlyGeometryNormals = 0;
    c->UseEnergyCompensation = 1; c->FurnaceTestMode = 0; c->MaxSamplesAccumulated = 5000; c->FramesInFlight = 0;
    return B200PT_OK;
}
int32_t b200pt_set_config(b200pt_handle h, const b200pt_config *c) { if (!c) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_config(*c); }); }
int32_t b200pt_get_config(b200pt_handle h, b200pt_config *c) { if (!c) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *c = e.config(); }); }
int32_t b200pt_material_count(b200pt_handle h, uint32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = (uint32_t)e.scene().materials.size(); }); }
int32_t b200pt_get_material(b200pt_handle h, uint32_t i, b200pt_material *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { if (i >= e.scene().materials.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "material index out of range" }; *out = e.scene().materials[i]; });
}
int32_t b200pt_set_material(b200pt_handle h, uint32_t i, const b200pt_material *m) { if (!m) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_material(i, *m); }); }
int32_t b200pt_get_material_name(b200pt_handle h, uint32_t i, char *buf, uint32_t n) {
    if (!buf || !n) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { if (i >= e.scene().material_names.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "material index out of range" };
        strncpy(buf, e.scene().material_names[i].c_str(), n - 1); buf[n - 1] = 0; });
}
int32_t b200pt_instance_count(b200pt_handle h, uint32_t *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { if (!e.has_scene()) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" }; *out = (uint32_t)e.scene().instances.size(); });
}
int32_t b200pt_get_instance_transforms(b200pt_handle h, float *xf, uint32_t count) {
    if (!xf) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        if (!e.has_scene()) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
        const auto &in = e.scene().instances;
        if (count != in.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "transform count differs from the instance count" };
        for (size_t i = 0; i < in.size(); i++) memcpy(xf + i * 16, in[i].Transform, sizeof in[i].Transform);
    });
}
int32_t b200pt_update_instance_transforms(b200pt_handle h, const float *xf, uint32_t count, int32_t rebuild) {
    if (!xf) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.update_instance_transforms(xf, count, rebuild); });
}
static const HostMesh &mesh_of(Engine &e, uint32_t mesh) {
    if (!e.has_scene()) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (mesh >= e.scene().meshes.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "mesh index out of range" };
    return e.scene().meshes[mesh];
}
int32_t b200pt_mesh_count(b200pt_handle h, uint32_t *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { if (!e.has_scene()) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" }; *out = (uint32_t)e.scene().meshes.size(); });
}
int32_t b200pt_mesh_vertex_count(b200pt_handle h, uint32_t mesh, uint32_t *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { *out = (uint32_t)mesh_of(e, mesh).vertices.size(); });
}
int32_t b200pt_get_mesh_vertices(b200pt_handle h, uint32_t mesh, b200pt_vertex *out, uint32_t count) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        const HostMesh &m = mesh_of(e, mesh);
        if (count != m.vertices.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "vertex count differs from the mesh's" };
        if (count) memcpy(out, m.vertices.data(), (size_t)count * sizeof(b200pt_vertex));
    });
}
int32_t b200pt_update_mesh_vertices(b200pt_handle h, const b200pt_mesh_update *updates, uint32_t n_updates, int32_t vertices_are_device, int32_t rebuild) {
    if (!updates || n_updates == 0) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.update_mesh_vertices(updates, n_updates, vertices_are_device != 0, rebuild); });
}
static const HostAnimation &animation_of(Engine &e) {
    if (!e.has_scene()) throw CudaError{ B200PT_ERR_NO_SCENE, "no scene" };
    if (!e.scene().animation) throw CudaError{ B200PT_ERR_NO_SCENE, "the scene has no glTF node data (loaded from OBJ or set through arrays)" };
    return *e.scene().animation;
}
static void copy_name(const std::string &s, char *buf, uint32_t n) { if (buf && n) { strncpy(buf, s.c_str(), n - 1); buf[n - 1] = 0; } }
int32_t b200pt_animation_count(b200pt_handle h, uint32_t *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { *out = (uint32_t)animation_of(e).clips.size(); });
}
int32_t b200pt_get_animation(b200pt_handle h, uint32_t index, char *name, uint32_t name_len, float *t0, float *t1) {
    return guard(h, [&](Engine &e) {
        const HostAnimation &a = animation_of(e);
        if (index >= a.clips.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "animation index out of range" };
        copy_name(a.clips[index].name, name, name_len);
        if (t0) *t0 = a.clips[index].t0;
        if (t1) *t1 = a.clips[index].t1;
    });
}
int32_t b200pt_pose(b200pt_handle h, int32_t animation, float time, int32_t rebuild) { return guard(h, [&](Engine &e) { e.pose(animation, time, rebuild); }); }
int32_t b200pt_set_camera(b200pt_handle h, const float vi[16], const float pi[16]) { if (!vi || !pi) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_camera(vi, pi); }); }
int32_t b200pt_get_camera(b200pt_handle h, float vi[16], float pi[16]) { if (!vi || !pi) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.get_camera(vi, pi); }); }
int32_t b200pt_camera_from_view(const float view[16], float aspect, float vi[16], float pi[16]) {
    if (!view || !vi || !pi || !(aspect > 0.0f)) return B200PT_ERR_WRONG_ARGUMENTS;
    camera_from_view(view, aspect, vi, pi); return B200PT_OK;
}
int32_t b200pt_resize(b200pt_handle h, uint32_t w, uint32_t hh) { return guard(h, [&](Engine &e) { e.resize(w, hh); }); }
int32_t b200pt_get_size(b200pt_handle h, uint32_t *w, uint32_t *hh) { if (!w || !hh) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *w = e.width(); *hh = e.height(); }); }
int32_t b200pt_reset(b200pt_handle h) { return guard(h, [&](Engine &e) { e.reset(); }); }
int32_t b200pt_default_volume(b200pt_volume *v) {                                      /* PT/PathTracer.h:36-70 */
    if (!v) return B200PT_ERR_WRONG_ARGUMENTS;
    memset(v, 0, sizeof *v);
    for (int k = 0; k < 3; k++) { v->CornerMin[k] = -1.0f; v->CornerMax[k] = 1.0f; v->Position[k] = 0.0f; v->Scale[k] = 1.0f; v->Color[k] = 0.8f; v->EmissiveColor[k] = 0.0f; }
    v->TemperatureColor[0] = 1.0f; v->TemperatureColor[1] = 0.5f; v->TemperatureColor[2] = 0.0f;
    v->Density = 1.0f; v->Anisotropy = 0.0f; v->Alpha = 1.0f; v->DropletSize = 20.0f; v->DensityDataIndex = -1; v->MaxDensityInTheGrid = 0.0f;
    v->UseBlackbody = 1; v->HasTemperatureData = 0; v->TemperatureGamma = 1.0f; v->TemperatureScale = 1.0f; v->EmissiveColorGamma = 1.0f;
    v->KelvinMin = 500; v->KelvinMax = 8000;
    v->ApproximatedScatteringForClouds = 0; v->ApproximatedScatteringFalloff = 0.8f; v->GridSharpness = 1.0f;
    return B200PT_OK;
}
int32_t b200pt_add_volume(b200pt_handle h, const b200pt_volume *v) { if (!v) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.add_volume(*v); }); }
int32_t b200pt_set_volume(b200pt_handle h, uint32_t i, const b200pt_volume *v) { if (!v) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_volume(i, *v); }); }
int32_t b200pt_remove_volume(b200pt_handle h, uint32_t i) { return guard(h, [&](Engine &e) { e.remove_volume(i); }); }
int32_t b200pt_volume_count(b200pt_handle h, uint32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = (uint32_t)e.volumes().size(); }); }
int32_t b200pt_get_volume(b200pt_handle h, uint32_t i, b200pt_volume *out) {
    if (!out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { if (i >= e.volumes().size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "volume index out of range" }; *out = e.volumes()[i]; });
}
int32_t b200pt_add_density_grid_to_volume(b200pt_handle h, uint32_t i, const b200pt_density_grid *g) { if (!g) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.add_density_grid(i, *g); }); }
int32_t b200pt_add_density_data_to_volume(b200pt_handle h, uint32_t, const char *) { if (h) h->err = "reading .vdb files needs OpenVDB (not in this build): read the grid with the reference's OpenVDB and call b200pt_add_density_grid_to_volume"; return B200PT_ERR_NOT_IMPLEMENTED; }
int32_t b200pt_remove_density_data_from_volume(b200pt_handle h, uint32_t i) { return guard(h, [&](Engine &e) { e.remove_density_data(i); }); }
int32_t b200pt_prepare_density_grid(const b200pt_density_grid *g, float *values, float *maxd, float cmin[3], float cmax[3], float *max_density) {
    if (!g || !values || !maxd || !cmin || !cmax || !max_density) return B200PT_ERR_WRONG_ARGUMENTS;
    try {
        PreparedGrid p; prepare_density_grid(*g, p);
        std::copy(p.values.begin(), p.values.end(), values); std::copy(p.max_densities.begin(), p.max_densities.end(), maxd);
        for (int k = 0; k < 3; k++) { cmin[k] = p.corner_min[k]; cmax[k] = p.corner_max[k]; }
        *max_density = p.max_density;
        return B200PT_OK;
    } catch (const CudaError &e) { return e.code; } catch (...) { return B200PT_ERR_UNKNOWN; }
}
static int32_t host_hook(const std::function<void()> &f) {       // the error text goes to b200pt_last_error(NULL)
    try { f(); return B200PT_OK; }
    catch (const CudaError &e) { g_err = e.what; return e.code < 0 ? e.code : B200PT_ERR_UNKNOWN; }
    catch (const std::bad_alloc &) { g_err = "host out of memory"; return B200PT_ERR_OUT_OF_MEMORY; }
    catch (...) { g_err = "unknown error"; return B200PT_ERR_UNKNOWN; }
}
static void load_for_hook(const char *path, HostScene &sc) {
    std::string err;
    if (!load_scene_file(path, sc, err)) throw CudaError{ B200PT_ERR_INIT_FAILED, "Failed to import scene: " + err };
    if (!sc.animation) throw CudaError{ B200PT_ERR_NO_SCENE, "the scene has no glTF node data" };
}
int32_t b200pt_gltf_animation_info(const char *path, int32_t index, uint32_t *count, char *name, uint32_t name_len, float *t0, float *t1) {
    if (!path || !count) return B200PT_ERR_WRONG_ARGUMENTS;
    return host_hook([&] {
        HostScene sc; load_for_hook(path, sc);
        const auto &clips = sc.animation->clips;
        *count = (uint32_t)clips.size();
        if (index < 0) return;
        if ((size_t)index >= clips.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "animation index out of range" };
        copy_name(clips[index].name, name, name_len);
        if (t0) *t0 = clips[index].t0;
        if (t1) *t1 = clips[index].t1;
    });
}
int32_t b200pt_gltf_pose_nodes(const char *path, int32_t animation, float time, uint32_t *node_count, float *world, uint32_t *weight_counts,
                               float *weights, uint32_t *weights_total) {
    if (!path || !node_count || !weights_total) return B200PT_ERR_WRONG_ARGUMENTS;
    return host_hook([&] {
        HostScene sc; load_for_hook(path, sc);
        const HostAnimation &a = *sc.animation;
        if (animation < -1 || animation >= (int)a.clips.size()) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "animation index out of range" };
        if (!std::isfinite(time)) throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "time is not finite" };
        HostPose P; evaluate_pose(a, sc, animation, time, P);
        *node_count = (uint32_t)P.world.size();
        size_t nw = 0; for (const auto &w : P.weights) nw += w.size();
        *weights_total = (uint32_t)nw;
        if (!world) return;
        for (size_t i = 0; i < P.world.size(); i++) m4_to_colmajor(P.world[i], world + i * 16);
        size_t o = 0;
        for (size_t i = 0; i < P.weights.size(); i++) {
            if (weight_counts) weight_counts[i] = (uint32_t)P.weights[i].size();
            if (weights) for (float x : P.weights[i]) weights[o++] = x;
        }
    });
}
int32_t b200pt_default_atmosphere(b200pt_atmosphere *a) {          // PathTracer.h:221-232
    if (!a) return B200PT_ERR_WRONG_ARGUMENTS;
    memset(a, 0, sizeof *a);
    a->Enable = 0; a->PlanetPosition[0] = 0.0f; a->PlanetPosition[1] = 6360e3f + 1000.0f; a->PlanetPosition[2] = 0.0f;
    a->PlanetRadius = 6360e3f; a->AtmosphereHeight = 100e3f;
    for (int k = 0; k < 3; k++) { a->RayleighScatteringCoefficientMultiplier[k] = 1.0f; a->MieScatteringCoefficientMultiplier[k] = 1.0f; a->OzoneAbsorptionCoefficientMultiplier[k] = 1.0f; }
    a->RayleighDensityFalloff = 8000.0f; a->MieDensityFalloff = 1200.0f; a->OzoneDensityFalloff = 5000.0f; a->OzonePeak = 22000.0f;
    a->SunColor[0] = 1.0f; a->SunColor[1] = 0.956f; a->SunColor[2] = 0.88f;
    return B200PT_OK;
}
int32_t b200pt_set_atmosphere(b200pt_handle h, const b200pt_atmosphere *a) {
    if (!a) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        if (!(a->PlanetRadius > 0.0f) || !(a->AtmosphereHeight >= 0.0f) || !(a->RayleighDensityFalloff > 0.0f) || !(a->MieDensityFalloff > 0.0f) || !(a->OzoneDensityFalloff > 0.0f))
            throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, "atmosphere: radius and density falloffs must be positive" };
        e.set_atmosphere(*a);
    });
}
int32_t b200pt_get_atmosphere(b200pt_handle h, b200pt_atmosphere *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.atmosphere(); }); }
int32_t b200pt_get_total_counts(b200pt_handle h, uint64_t *nv, uint64_t *ni) {
    if (!nv || !ni) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { uint64_t v = 0, i = 0; for (const auto &m : e.scene().meshes) { v += m.vertices.size(); i += m.indices.size(); } *nv = v; *ni = i; });
}
int32_t b200pt_set_phase_function(b200pt_handle h, uint32_t pf) { return guard(h, [&](Engine &e) { e.set_phase_function(pf); }); }
int32_t b200pt_get_phase_function(b200pt_handle h, uint32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.phase_function(); }); }

int32_t b200pt_set_partition(b200pt_handle h, uint32_t r, uint32_t w, uint32_t b) { return guard(h, [&](Engine &e) { e.set_partition(r, w, b); }); }
int32_t b200pt_local_rows(b200pt_handle h, uint32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.local_rows(); }); }
uint32_t b200pt_partition_global_row(uint32_t lr, uint32_t r, uint32_t w, uint32_t b) { return partition_global_row(lr, r, w, b); }
uint32_t b200pt_partition_local_row_count(uint32_t H, uint32_t r, uint32_t w, uint32_t b) { return partition_local_rows(H, r, w, b); }

int32_t b200pt_path_trace(b200pt_handle h, uint32_t dispatches, uint32_t seed, int32_t *done) {
    return guard(h, [&](Engine &e) { bool d = e.path_trace(dispatches, seed); if (done) *done = d ? 1 : 0; });
}
int32_t b200pt_default_adaptive(b200pt_adaptive *a) {
    if (!a) return B200PT_ERR_WRONG_ARGUMENTS;
    a->Enable = 0; a->Threshold = 0.01f; a->MinSamples = 64; a->Interval = 32;
    return B200PT_OK;
}
int32_t b200pt_set_adaptive(b200pt_handle h, const b200pt_adaptive *a) { if (!a) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_adaptive(*a); }); }
int32_t b200pt_get_adaptive(b200pt_handle h, b200pt_adaptive *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.adaptive(); }); }
int32_t b200pt_get_pixel_stats(b200pt_handle h, uint32_t *counts, float *rel_error) { return guard(h, [&](Engine &e) { e.pixel_stats(counts, rel_error); }); }
int32_t b200pt_set_track_variance(b200pt_handle h, int32_t enable) { return guard(h, [&](Engine &e) { e.set_track_variance(enable != 0); }); }
int32_t b200pt_get_track_variance(b200pt_handle h, int32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.track_variance() ? 1 : 0; }); }
int32_t b200pt_default_denoise(b200pt_denoise_params *p) {
    if (!p) return B200PT_ERR_WRONG_ARGUMENTS;
    p->Iterations = 5; p->FeatureSamples = 8; p->SigmaLuminance = 4.0f; p->SigmaNormal = 128.0f; p->SigmaDepth = 1.0f;
    return B200PT_OK;
}
int32_t b200pt_denoise(b200pt_handle h, const b200pt_denoise_params *p, float *elapsed_ms) {
    if (!p) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.denoise(*p, elapsed_ms); });
}
int32_t b200pt_get_denoised(b200pt_handle h, float *dst, int32_t dev) { if (!dst) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.get_denoised(dst, dev != 0); }); }
int32_t b200pt_get_denoise_inputs(b200pt_handle h, const b200pt_denoise_params *p, float *albedo_cov, float *normal_depth, float *variance) {
    if (!p) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.denoise_inputs(*p, albedo_cov, normal_depth, variance); });
}
int32_t b200pt_denoise_image(b200pt_handle h, uint32_t w, uint32_t ht, const float *color, const float *albedo_cov, const float *normal_depth,
                             const float *variance, const b200pt_denoise_params *p, float *out, int32_t dev) {
    if (!color || !albedo_cov || !normal_depth || !variance || !p || !out) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.denoise_image(w, ht, color, albedo_cov, normal_depth, variance, *p, out, dev != 0); });
}
int32_t b200pt_post_process_denoised(b200pt_handle h) { return guard(h, [&](Engine &e) { e.post_process_denoised(); }); }
int32_t b200pt_active_pixels(b200pt_handle h, uint32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.active_pixels(); }); }
int32_t b200pt_flush(b200pt_handle h) { return guard(h, [&](Engine &e) { e.flush(); }); }
int32_t b200pt_samples_accumulated(b200pt_handle h, uint32_t *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.samples_accumulated(); }); }
int32_t b200pt_synchronize(b200pt_handle h) { return guard(h, [&](Engine &e) { e.synchronize(); }); }
int32_t b200pt_set_stream(b200pt_handle h, void *s) { return guard(h, [&](Engine &e) { e.set_stream((cudaStream_t)s); }); }
int32_t b200pt_set_profiling(b200pt_handle h, int32_t on) { return guard(h, [&](Engine &e) { e.set_profiling(on != 0); }); }
int32_t b200pt_get_hdr(b200pt_handle h, float *dst, int32_t dev) { if (!dst) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.get_hdr(dst, dev != 0); }); }
int32_t b200pt_hdr_device_ptr(b200pt_handle h, void **out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.synchronize(); *out = e.hdr_device(); }); }
int32_t b200pt_set_hdr(b200pt_handle h, const float *src, int32_t dev) { if (!src) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_hdr(src, dev != 0); }); }
int32_t b200pt_save_checkpoint(b200pt_handle h, const char *path) { if (!path) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.save_checkpoint(path); }); }
int32_t b200pt_load_checkpoint(b200pt_handle h, const char *path) { if (!path) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.load_checkpoint(path); }); }
int32_t b200pt_get_counters(b200pt_handle h, b200pt_counters *out) { if (!out) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { *out = e.counters(); }); }

int32_t b200pt_post_set_tonemap(b200pt_handle h, const b200pt_tonemap *t) { if (!t) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_tonemap(*t); }); }
int32_t b200pt_post_set_bloom(b200pt_handle h, const b200pt_bloom *b) { if (!b) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.set_bloom(*b); }); }
int32_t b200pt_post_process(b200pt_handle h) { return guard(h, [&](Engine &e) { e.post_process(); }); }
int32_t b200pt_accumulate_rows(b200pt_handle h, const float *frame_device, uint32_t frame_index, uint32_t y0, uint32_t y1) {
    return guard(h, [&](Engine &e) { e.accumulate_rows(reinterpret_cast<const float4 *>(frame_device), frame_index, y0, y1); });
}
int32_t b200pt_post_input_rows(b200pt_handle h, uint32_t y0, uint32_t y1, uint32_t *in0, uint32_t *in1) {
    if (!in0 || !in1) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.post_input_rows(y0, y1, in0, in1); });
}
int32_t b200pt_post_process_rows(b200pt_handle h, uint32_t y0, uint32_t y1) { return guard(h, [&](Engine &e) { e.post_process_rows(y0, y1); }); }
int32_t b200pt_get_ldr_rows(b200pt_handle h, uint32_t y0, uint32_t y1, uint8_t *dst, int32_t dev) { return guard(h, [&](Engine &e) { e.get_ldr_rows(y0, y1, dst, dev != 0); }); }
int32_t b200pt_get_ldr(b200pt_handle h, uint8_t *dst, int32_t dev) { if (!dst) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.get_ldr(dst, dev != 0); }); }
int32_t b200pt_get_bloom(b200pt_handle h, float *dst) { if (!dst) return B200PT_ERR_WRONG_ARGUMENTS; return guard(h, [&](Engine &e) { e.get_bloom(dst); }); }
int32_t b200pt_bloom_mip_sizes(uint32_t w, uint32_t hh, uint32_t *wh, uint32_t *levels) { if (!wh || !levels || !w || !hh) return B200PT_ERR_WRONG_ARGUMENTS; *levels = bloom_mip_sizes(w, hh, wh); return B200PT_OK; }
int32_t b200pt_save_png(b200pt_handle h, const char *path) {     // Editor::SaveToFile (Editor.cpp:815-843)
    if (!path) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        std::vector<uint8_t> px((size_t)e.width() * e.height() * 4);
        e.get_ldr(px.data(), false);
        if (!write_png_rgba8(path, e.width(), e.height(), px.data())) throw CudaError{ B200PT_ERR_UNKNOWN, std::string("cannot write ") + path };
    });
}

int32_t b200pt_volume_walks(b200pt_handle h, uint32_t n, const float *o, const float *d, const uint32_t *seeds, float depth, float *T, float *sd, int32_t *vol, uint32_t *rng2) {
    if (n && (!o || !d || !seeds || !T || !sd || !vol || !rng2)) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.volume_walks(n, o, d, seeds, depth, T, sd, vol, rng2); });
}
int32_t b200pt_trace_closest(b200pt_handle h, uint32_t n, const float *o, const float *d, float tmin, float tmax, float *t, uint32_t *prim, uint32_t *inst, float *uv) {
    if (n && (!o || !d || !t || !prim || !inst || !uv)) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.trace_closest(n, o, d, tmin, tmax, t, prim, inst, uv); });
}
int32_t b200pt_trace_stats(b200pt_handle h, uint32_t n, const float *o, const float *d, float tmin, float tmax, uint32_t *nodes_tris) {
    if (n && (!o || !d || !nodes_tris)) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { std::vector<float> t(n), uv(2 * (size_t)n); std::vector<uint32_t> p(n), i(n); e.trace_closest(n, o, d, tmin, tmax, t.data(), p.data(), i.data(), uv.data(), nodes_tris); });
}
int32_t b200pt_trace_query(b200pt_handle h, int32_t shape, int32_t kind, int32_t fma_slabs, uint32_t n, const float *o, const float *d, const float *tmin,
                           const float *tmax, const uint32_t *target, const float *tmax_test, float *t, uint32_t *prim, uint32_t *inst, float *uv,
                           uint32_t *occluded, uint32_t *stats) {
    if (shape < 0 || shape >= TQ_SHAPES || kind < TQ_CLOSEST || kind > TQ_TARGET) return B200PT_ERR_WRONG_ARGUMENTS;
    if (n && (!o || !d || !tmin || !tmax || (kind == TQ_TARGET && (!target || !tmax_test)) || (kind == TQ_CLOSEST ? (!t || !prim || !inst || !uv) : !occluded)))
        return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.trace_query(shape, kind, fma_slabs != 0, n, o, d, tmin, tmax, target, tmax_test, t, prim, inst, uv, occluded, stats); });
}
int32_t b200pt_shade_query(b200pt_handle h, int32_t force_general, uint32_t n, const uint32_t *inst, const uint32_t *prim, const float *uv, const float *d,
                           const float *o, const float *pay_pdf, const uint32_t *rng, const float *L, float *out) {
    if (n && (!inst || !prim || !uv || !d || !o || !pay_pdf || !rng || !out)) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.shade_query(force_general != 0, n, inst, prim, uv, d, o, pay_pdf, rng, L, out); });
}
int32_t b200pt_miss_query(b200pt_handle h, uint32_t n, const float *d, const uint32_t *depth, const float *pay_pdf, float *out) {
    if (n && (!d || !depth || !pay_pdf || !out)) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.miss_query(n, d, depth, pay_pdf, out); });
}
int32_t b200pt_bounce_query(b200pt_handle h, uint32_t n, const float *in, uint32_t flags, float *out, uint32_t *survivors) {
    if (!survivors || (n && (!in || !out))) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.bounce_query(n, in, flags, out, survivors); });
}
int32_t b200pt_bake_lut(b200pt_handle h, int32_t kind, uint32_t sx, uint32_t sy, uint32_t sz, uint32_t sample_count, uint32_t seed, uint32_t slices, float *out, float *elapsed_ms) {
    if (!out || kind < 0 || kind > 2 || !sx || !sy || !sz) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) { e.bake_lut(kind, sx, sy, sz, sample_count, seed, slices, out, elapsed_ms); });
}
// Application.cpp:35-72: bake the three tables with the reference's sizes and write the .bin files that are missing in `dir`.
int32_t b200pt_bake_luts_to_dir(b200pt_handle h, const char *dir, uint32_t sample_count, uint32_t seed, int32_t overwrite) {
    if (!dir) return B200PT_ERR_WRONG_ARGUMENTS;
    static const struct { const char *name; int kind; uint32_t sx, sy, sz; } tabs[3] = {
        { "ReflectionLookup.bin", 0, 64, 64, 32 }, { "RefractionLookupHitFromOutside.bin", 1, 128, 128, 32 }, { "RefractionLookupHitFromInside.bin", 2, 128, 128, 32 } };
    for (const auto &t : tabs) {
        const std::string path = std::string(dir) + "/" + t.name;
        if (!overwrite) { FILE *f = fopen(path.c_str(), "rb"); if (f) { fclose(f); continue; } }
        std::vector<float> data((size_t)t.sx * t.sy * t.sz);
        int32_t r = guard(h, [&](Engine &e) { e.bake_lut(t.kind, t.sx, t.sy, t.sz, sample_count, seed, 0, data.data(), nullptr); });
        if (r != B200PT_OK) return r;
        FILE *f = fopen(path.c_str(), "wb");
        if (!f) { g_err = "cannot write " + path; return B200PT_ERR_INIT_FAILED; }
        const size_t w = fwrite(data.data(), sizeof(float), data.size(), f); fclose(f);
        if (w != data.size()) { g_err = "short write " + path; return B200PT_ERR_UNKNOWN; }
    }
    return B200PT_OK;
}
int32_t b200pt_scene_stats(b200pt_handle h, uint32_t *a, uint32_t *b, uint32_t *c, uint32_t *d) { return guard(h, [&](Engine &e) { e.scene_stats(a, b, c, d); }); }

// ---- standalone codecs ----
int32_t b200pt_decode_image_file(const char *path, uint32_t *w, uint32_t *hh, uint8_t **out) {
    if (!path || !w || !hh || !out) return B200PT_ERR_WRONG_ARGUMENTS;
    std::vector<uint8_t> px; std::string err;
    try { if (!decode_image_rgba8(path, *w, *hh, px, err)) { g_err = err; return B200PT_ERR_INIT_FAILED; } }   // no exception crosses the boundary (Error.h:14-72)
    catch (const std::bad_alloc &) { g_err = "out of memory while decoding " + std::string(path); return B200PT_ERR_OUT_OF_MEMORY; }
    catch (...) { g_err = "unexpected failure while decoding " + std::string(path); return B200PT_ERR_UNKNOWN; }
    *out = (uint8_t *)malloc(px.size() ? px.size() : 1); if (!*out) return B200PT_ERR_OUT_OF_MEMORY;
    memcpy(*out, px.data(), px.size()); return B200PT_OK;
}
int32_t b200pt_decode_hdr_file(const char *path, uint32_t *w, uint32_t *hh, float **out) {
    if (!path || !w || !hh || !out) return B200PT_ERR_WRONG_ARGUMENTS;
    std::vector<float> px; std::string err;
    try { if (!decode_hdr_rgba32f(path, *w, *hh, px, err)) { g_err = err; return B200PT_ERR_INIT_FAILED; } }
    catch (const std::bad_alloc &) { g_err = "out of memory while decoding " + std::string(path); return B200PT_ERR_OUT_OF_MEMORY; }
    catch (...) { g_err = "unexpected failure while decoding " + std::string(path); return B200PT_ERR_UNKNOWN; }
    *out = (float *)malloc(px.size() ? px.size() * 4 : 4); if (!*out) return B200PT_ERR_OUT_OF_MEMORY;
    memcpy(*out, px.data(), px.size() * 4); return B200PT_OK;
}
int32_t b200pt_write_png(const char *path, uint32_t w, uint32_t hh, const uint8_t *rgba) {
    if (!path || !w || !hh || !rgba) return B200PT_ERR_WRONG_ARGUMENTS;
    return write_png_rgba8(path, w, hh, rgba) ? B200PT_OK : B200PT_ERR_UNKNOWN;
}
int32_t b200pt_bvh4_collapse(const void *nodes2, uint32_t n_nodes2, int32_t root2, void *nodes4_out, uint32_t *n_nodes4_out, int32_t *depth_out) {
    if (!nodes2 || !nodes4_out || !n_nodes4_out || !n_nodes2) return B200PT_ERR_WRONG_ARGUMENTS;
    if (root2 >= 0 && (uint32_t)root2 >= n_nodes2) return B200PT_ERR_WRONG_ARGUMENTS;
    int d = 0;
    *n_nodes4_out = b200pt::bvh4_collapse_host(static_cast<const b200pt::BvhNode *>(nodes2), n_nodes2, root2, static_cast<b200pt::Bvh4Node *>(nodes4_out), &d);
    if (depth_out) *depth_out = d;
    return B200PT_OK;
}
int32_t b200pt_bvh2_sah_rebuild(const void *nodes2, uint32_t n_nodes2, int32_t root2, void *out, uint32_t *n_out, int32_t *depth_out, double *sah) {
    if (!nodes2 || !out || !n_out || !n_nodes2) return B200PT_ERR_WRONG_ARGUMENTS;
    if (root2 >= 0 && (uint32_t)root2 >= n_nodes2) return B200PT_ERR_WRONG_ARGUMENTS;
    int d = 0; double c[2] = { 0.0, 0.0 };
    try { *n_out = b200pt::bvh2_sah_rebuild_host(static_cast<const b200pt::BvhNode *>(nodes2), n_nodes2, root2, static_cast<b200pt::BvhNode *>(out), &d, c); }
    catch (...) { return B200PT_ERR_OUT_OF_MEMORY; }
    if (depth_out) *depth_out = d;
    if (sah) { sah[0] = c[0]; sah[1] = c[1]; }
    return B200PT_OK;
}
int32_t b200pt_bvh2_sah_build(const float *ref_boxes, uint32_t n, float trav_cost, void *out, uint32_t *perm, uint32_t *n_out, int32_t *depth_out, double *sah_cost) {
    if (!ref_boxes || !out || !perm || !n_out || !n || !(trav_cost >= 0.0f)) return B200PT_ERR_WRONG_ARGUMENTS;
    int d = 0; double c = 0.0;
    try { *n_out = b200pt::bvh2_sah_build_host(ref_boxes, n, trav_cost, static_cast<b200pt::BvhNode *>(out), perm, &d, &c); }
    catch (...) { return B200PT_ERR_OUT_OF_MEMORY; }
    if (depth_out) *depth_out = d;
    if (sah_cost) *sah_cost = c;
    return B200PT_OK;
}
int32_t b200pt_bvh2_ploc_build(const float *ref_boxes, uint32_t n, void *out, uint32_t *perm, uint32_t *n_out, int32_t *depth_out, double *sah_cost) {
    if (!ref_boxes || !out || !perm || !n_out || !n) return B200PT_ERR_WRONG_ARGUMENTS;
    int d = 0; double c = 0.0;
    try { *n_out = b200pt::bvh2_ploc_build_host(ref_boxes, n, static_cast<b200pt::BvhNode *>(out), perm, &d, &c); }
    catch (...) { return B200PT_ERR_OUT_OF_MEMORY; }
    if (depth_out) *depth_out = d;
    if (sah_cost) *sah_cost = c;
    return B200PT_OK;
}
int32_t b200pt_bvh2_ploc_build_query(b200pt_handle h, const float *ref_boxes, uint32_t n, void *nodes_out, uint32_t *perm_out, uint32_t *n_out, int32_t *depth_out,
                                     void *nodes4_out, uint32_t *n4_out, int32_t *depth4_out) {
    if (!ref_boxes || !nodes_out || !perm_out || !n_out || !nodes4_out || !n4_out || !n) return B200PT_ERR_WRONG_ARGUMENTS;
    return guard(h, [&](Engine &e) {
        int d = 0, d4 = 0;
        e.ploc_build_query(ref_boxes, n, static_cast<b200pt::BvhNode *>(nodes_out), perm_out, n_out, &d, static_cast<b200pt::Bvh4Node *>(nodes4_out), n4_out, &d4);
        if (depth_out) *depth_out = d;
        if (depth4_out) *depth4_out = d4;
    });
}
int32_t b200pt_bvh2_reinsert(const void *nodes2, uint32_t n_nodes2, int32_t root2, void *out, int32_t passes, float fraction, uint32_t *n_out, int32_t *depth_out, double *sah) {
    if (!nodes2 || !out || !n_out || !n_nodes2 || passes < 0 || passes > 64 || !(fraction >= 0.0f && fraction <= 1.0f)) return B200PT_ERR_WRONG_ARGUMENTS;
    if (root2 >= 0 && (uint32_t)root2 >= n_nodes2) return B200PT_ERR_WRONG_ARGUMENTS;
    int d = 0; double c[2] = { 0.0, 0.0 };
    try { *n_out = b200pt::bvh2_reinsert_host(static_cast<const b200pt::BvhNode *>(nodes2), n_nodes2, root2, static_cast<b200pt::BvhNode *>(out), passes, fraction, &d, c); }
    catch (...) { return B200PT_ERR_OUT_OF_MEMORY; }
    if (depth_out) *depth_out = d;
    if (sah) { sah[0] = c[0]; sah[1] = c[1]; }
    return B200PT_OK;
}
int32_t b200pt_build_env_alias(float *rgba, uint32_t w, uint32_t hh, void *alias, float *sum) {
    if (!rgba || !w || !hh || !alias) return B200PT_ERR_WRONG_ARGUMENTS;
    float s = build_env_alias(rgba, w, hh, (uint2 *)alias); if (sum) *sum = s; return B200PT_OK;
}

struct OwnedScene { b200pt_scene_desc desc; HostScene host; std::vector<b200pt_mesh> meshes; std::vector<b200pt_texture> textures; };
int32_t b200pt_load_gltf(const char *path, b200pt_scene_desc **out) {
    if (!path || !out) return B200PT_ERR_WRONG_ARGUMENTS;
    *out = nullptr;
    OwnedScene *o = new (std::nothrow) OwnedScene(); if (!o) return B200PT_ERR_OUT_OF_MEMORY;
    std::string err;
    try {
        if (!load_scene_file(path, o->host, err)) { g_err = err; delete o; return B200PT_ERR_INIT_FAILED; }
        for (auto &m : o->host.meshes) o->meshes.push_back({ m.vertices.data(), m.indices.data(), (uint32_t)m.vertices.size(), (uint32_t)m.indices.size() });
        for (auto &t : o->host.textures) o->textures.push_back({ t.width, t.height, t.channels, 0, t.data.data() });
    } catch (const std::bad_alloc &) { delete o; g_err = "out of memory while importing the scene"; return B200PT_ERR_OUT_OF_MEMORY; }
    catch (...) { delete o; g_err = "unexpected failure while importing the scene"; return B200PT_ERR_UNKNOWN; }
    memset(&o->desc, 0, sizeof o->desc);
    o->desc.meshes = o->meshes.data(); o->desc.mesh_count = (uint32_t)o->meshes.size();
    o->desc.materials = o->host.materials.data(); o->desc.material_count = (uint32_t)o->host.materials.size();
    o->desc.textures = o->textures.data(); o->desc.texture_count = (uint32_t)o->textures.size();
    o->desc.instances = o->host.instances.data(); o->desc.instance_count = (uint32_t)o->host.instances.size();
    memcpy(o->desc.camera_view, o->host.camera_view, sizeof o->desc.camera_view); o->desc.camera_aspect = o->host.camera_aspect;
    *out = &o->desc;     // desc is the first member: the pointer doubles as the owner
    return B200PT_OK;
}
int32_t b200pt_free_scene(b200pt_scene_desc *s) { if (!s) return B200PT_ERR_WRONG_ARGUMENTS; delete reinterpret_cast<OwnedScene *>(s); return B200PT_OK; }
void b200pt_free(void *p) { free(p); }

} // extern "C"
