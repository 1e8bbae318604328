// Host-only check that the host runtime leaves no CUDA resource behind on any error path.  The runtime calls that create, copy and
// release are replaced by shims defined in THIS file (the executable's own symbols win over libcudart's, as in refine_plumbing.cpp):
// device and pinned memory are zeroed host blocks, events and streams are host blocks as well, every live one is tracked, kernel
// launches do nothing, and a device-to-host copy fills its destination with a chosen word (what the builders read back).  For every k:
//   * Engine (b200pt_create): the k-th creation of a stream, event or block fails; nothing is live after the error, nor after
//     b200pt_destroy of an engine whose creation succeeded;
//   * lbvh_build, ploc_build, lbvh_ploc_rebuild, bvh4_collapse_device, lbvh_build_wide, lbvh_build_wide_device: the k-th cudaMalloc
//     fails; a failing call leaves nothing live, a successful call exactly its outputs;
//   * the first lbvh_refit of a tree, with and without a BVH4: the k-th cudaMalloc of the refit state fails; a failing call leaves the
//     tree and no refit state, the next call succeeds, and a successful call leaves exactly the tree and its refit state;
//   * lbvh_build of a scene whose split counts add up to 2^28 references returns an error and leaves nothing live;
//   * Engine::set_env_map, set_luts and set_material (its emissive rebuild) on an engine with a scene, a map and tables: the k-th creation
//     fails; every non-null pointer of the device view (Engine::dev_scene) lies in a live block and has_env / has_luts agree with it.  A
//     failed set_env_map / set_luts leaves no map / no tables, and every launch that reads them refuses with B200PT_ERR_NO_SCENE; a failed
//     emissive rebuild leaves the previous tables; a successful call leaves exactly its new blocks, and the view holds them.
// The trees handed to the functions under test are blocks of the shim too, so the LbvhResult that owns them releases them.  query_launch_cfg's
// device queries (set_scene) are shims as well.
// Built and run by tests/test_resource_ownership.py: nvcc --cudart shared ... tests/native/alloc_faults.cpp <every object of build/> -lz
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <vector>
#include <cuda_runtime.h>
#include "kernels.h"
#include "engine.h"
#include "b200pt.h"
using namespace b200pt;

static long g_fail_at = 0, g_created = 0;      // creations since the last arm(); the g_fail_at-th fails (0: none)
static std::set<void *> g_live;
struct Block { size_t bytes; long serial; };
static std::map<const char *, Block> g_blocks;  // every live block, with its size and its creation's number
static long g_serial = 0;
static uint32_t g_readback = 0;

static void arm(long k, uint32_t readback) { g_fail_at = k; g_created = 0; g_readback = readback; }
// Runs f with no creation failing and none counted: the inputs a case creates for the function under test.
template <class F> static void unarmed(F f) { const long k = g_fail_at, c = g_created; g_fail_at = 0; f(); g_fail_at = k; g_created = c; }
static cudaError_t create(void **p, size_t bytes) {
    *p = nullptr;
    if (++g_created == g_fail_at) return cudaErrorMemoryAllocation;
    *p = calloc(1, bytes ? bytes : 1);
    g_live.insert(*p); g_blocks[static_cast<const char *>(*p)] = { bytes ? bytes : 1, ++g_serial };
    return cudaSuccess;
}
static cudaError_t release(void *p) {
    if (!p) return cudaSuccess;
    if (!g_live.erase(p)) { printf("FAIL: release of a handle that is not live\n"); exit(1); }
    g_blocks.erase(static_cast<const char *>(p));
    free(p);
    return cudaSuccess;
}
// p points into a live block
static bool live(const void *p) {
    const char *c = static_cast<const char *>(p);
    auto it = g_blocks.upper_bound(c);
    if (it == g_blocks.begin()) return false;
    --it;
    return c < it->first + it->second.bytes;
}
static cudaError_t copy(void *dst, const void *src, size_t n, cudaMemcpyKind kind) {
    if (kind == cudaMemcpyDeviceToHost) for (size_t i = 0; i + 4 <= n; i += 4) memcpy(static_cast<char *>(dst) + i, &g_readback, 4);
    else memcpy(dst, src, n);
    return cudaSuccess;
}

extern "C" {
cudaError_t cudaMalloc(void **p, size_t n) { return create(p, n); }
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { return create(p, n); }
cudaError_t cudaFree(void *p) { return release(p); }
cudaError_t cudaFreeHost(void *p) { return release(p); }
cudaError_t cudaEventCreate(cudaEvent_t *e) { return create(reinterpret_cast<void **>(e), 1); }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return create(reinterpret_cast<void **>(e), 1); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { return release(e); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { return create(reinterpret_cast<void **>(s), 1); }
cudaError_t cudaStreamDestroy(cudaStream_t s) { return release(s); }
cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaGetLastError() { return cudaSuccess; }
cudaError_t cudaMemset(void *p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind k) { return copy(d, s, n, k); }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind k, cudaStream_t) { return copy(d, s, n, k); }
cudaError_t cudaLaunchKernel(const void *, dim3, dim3, void **, size_t, cudaStream_t) { return cudaSuccess; }
// what query_launch_cfg asks of the device when set_scene builds a tree: one CTA of every kernel per SM on 132 SMs
cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { memset(p, 0, sizeof *p); p->multiProcessorCount = 132; return cudaSuccess; }
cudaError_t cudaFuncGetAttributes(cudaFuncAttributes *a, const void *) { memset(a, 0, sizeof *a); return cudaSuccess; }
cudaError_t cudaFuncSetAttribute(const void *, cudaFuncAttribute, int) { return cudaSuccess; }
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, const void *, int, size_t) { *n = 1; return cudaSuccess; }
}

static int failures = 0;
static void expect(bool ok, const char *what, long k) { if (!ok) { printf("FAIL: %s (k = %ld)\n", what, k); failures++; } }

// Calls f for k = 1, 2, ... until a call creates fewer than k resources.  f returns its error code and, on success, the resources it
// hands to the caller (released here).  Prints "<name>: <creations> creations, <failed checks> failed".
template <class F> static void each_k(const char *name, uint32_t readback, bool must_succeed, F f) {
    const int failures0 = failures;
    for (long k = 1;; k++) {
        const std::set<void *> before = g_live;
        arm(k, readback);
        std::vector<void *> outputs;
        const int r = f(&outputs);
        const bool injected = g_created >= k;
        arm(0, readback);
        if (r != 0) expect(g_live == before, name, k);
        else {
            std::set<void *> want = before;
            for (void *p : outputs) if (p) want.insert(p);
            expect(!injected, "success although a creation failed", k);
            expect(g_live == want, name, k);
            for (void *p : outputs) release(p);
        }
        if (!injected) {
            expect(r == 0 || !must_succeed, name, k);
            printf("%s: %ld creations, %d failed\n", name, k - 1, failures - failures0);
            return;
        }
    }
}

int main() {
    // Engine: b200pt_create fails at every creation, then succeeds and is destroyed
    each_k("engine", 0, true, [](std::vector<void *> *) {
        b200pt_handle h = nullptr;
        const int r = b200pt_create(0, &h);
        if (r == B200PT_OK) b200pt_destroy(h);
        else if (h) { printf("FAIL: a handle despite the error\n"); failures++; }
        return r;
    });

    // lbvh_build: every triangle one reference (split counts read back as 1), reference boxes kept for both the host and the device builder
    const uint32_t nt = 1000;
    std::vector<b200pt_vertex> verts(3 * nt); std::vector<uint32_t> idx(3 * nt); DevMesh mesh{ 0, 0, nt, 0 }; DevInstance inst{};
    for (uint32_t i = 0; i < 3 * nt; i++) idx[i] = i;
    auto build = [&](uint32_t n_tris, std::vector<void *> *outs) {
        LbvhResult res{}; std::vector<float> host_ref_box; DevPtr<float> ref_box;
        const int r = lbvh_build(verts.data(), idx.data(), &mesh, &inst, 1, n_tris, &res, nullptr, &host_ref_box, &ref_box);
        if (r == 0) *outs = { res.shade.release(), res.tri_slot.release(), res.nodes.release(), ref_box.release() };
        return r;
    };
    each_k("lbvh_build", 1u, true, [&](std::vector<void *> *o) { return build(nt, o); });
    each_k("lbvh_build (2^28 references)", 1u << 20, false, [&](std::vector<void *> *o) {
        const int r = build(256, o);
        if (r == 0) { printf("FAIL: 2^28 references accepted\n"); failures++; }
        return r;
    });

    // the device tree builder and collapse on host arrays: one clustering step (cluster count read back as 1), one BVH4 level (0)
    std::vector<float> boxes((size_t)nt * 6, 0.0f); std::vector<BvhNode> nodes(nt - 1), nodes2(nt - 1); std::vector<uint32_t> perm(nt);
    std::vector<Bvh4Node> nodes4(nt - 1);
    // a tree of n_nodes zeroed nodes followed by n_tris slots, created through the shim and owned by the result
    auto tree = [](LbvhResult *res, uint32_t n_nodes, uint32_t n_tris) {
        unarmed([&] {
            alloc(res->nodes, (size_t)n_nodes * sizeof(BvhNode) + (size_t)n_tris * sizeof(BvhTri));
            alloc(res->tri_slot, (size_t)n_tris * 4);
        });
        res->tris = reinterpret_cast<BvhTri *>(res->nodes.get() + n_nodes); res->n_nodes = n_nodes; res->n_tris = res->n_prims = n_tris;
    };
    each_k("ploc_build", 1u, true, [&](std::vector<void *> *) {
        uint32_t n_out = 0; int depth = 0; uint32_t h_small[4];
        return ploc_build(boxes.data(), nt, nodes.data(), perm.data(), &n_out, &depth, h_small, nullptr);
    });
    each_k("lbvh_ploc_rebuild", 1u, true, [&](std::vector<void *> *) {
        LbvhResult res{}; tree(&res, nt - 1, nt); res.max_depth = 10;
        DevPtr<float> ref_box; unarmed([&] { alloc(ref_box, (size_t)nt * 6 * sizeof(float)); });   // from the caller, beside the tree
        uint32_t h_small[4];
        return lbvh_ploc_rebuild(&res, std::move(ref_box), h_small, nullptr);
    });
    each_k("bvh4_collapse_device", 0u, true, [&](std::vector<void *> *) {
        uint32_t n4 = 0, h_total[4]; int d4 = 0;
        return bvh4_collapse_device(nodes2.data(), nt - 1, 0, nodes4.data(), &n4, &d4, h_total, nullptr);
    });
    each_k("lbvh_build_wide_device", 0u, true, [&](std::vector<void *> *o) {
        LbvhResult res{}; tree(&res, nt - 1, 0);
        uint32_t h_small[4];
        const int r = lbvh_build_wide_device(&res, h_small, nullptr);
        *o = { res.nodes4.release() };
        return r;
    });
    // the host collapse: both children of the root read back as one-slot leaves (0xFFFFFFFF), one BVH4 node
    each_k("lbvh_build_wide", 0xFFFFFFFFu, true, [&](std::vector<void *> *o) {
        LbvhResult res{}; tree(&res, 1, 0);
        const int r = lbvh_build_wide(&res, nullptr);
        if (r == 0 && res.n_nodes4 != 1) { printf("FAIL: lbvh_build_wide made %u nodes\n", res.n_nodes4); failures++; }
        *o = { res.nodes4.release() };
        return r;
    });

    // the first refit of a tree derives its refit state: one root over two one-slot leaves (read back as 0xFFFFFFFF), four slots of one
    // triangle, and with `wide` a one-node BVH4
    auto refit = [&](bool wide) {
        LbvhResult res{}; tree(&res, 1, 4);
        if (wide) { unarmed([&] { alloc(res.nodes4, sizeof(Bvh4Node)); }); res.n_nodes4 = 1; }
        const long k = g_fail_at;
        const std::set<void *> tree_blocks = g_live;
        auto call = [&] { return lbvh_refit(&res, verts.data(), idx.data(), &mesh, &inst, 1, nullptr); };
        const LbvhRefit &s = res.refit;
        const int r = call();
        if (r != 0) {
            expect(g_live == tree_blocks && !s.ready && !s.slot_jk && !s.slot_box && !s.node_box && !s.bounds && !s.order && !s.src4 && s.level_off.empty(),
                   "failed refit: the tree and no refit state", k);
            int again = -1; unarmed([&] { again = call(); });
            expect(again == 0 && s.ready, "refit after a failed prepare", k);
        } else {
            std::set<void *> want = tree_blocks;
            for (void *p : std::initializer_list<void *>{ s.slot_jk.get(), s.slot_box.get(), s.node_box.get(), s.bounds.get(), s.order.get(), s.src4.get() })
                if (p) want.insert(p);
            expect(s.ready && s.slot_jk && s.slot_box && s.node_box && s.bounds && s.order && (s.src4 != nullptr) == wide && g_live == want,
                   "refit: the tree and its refit state", k);
        }
        return r;                                                  // res releases the tree and its refit state
    };
    each_k("lbvh_refit", 0xFFFFFFFFu, true, [&](std::vector<void *> *) { return refit(false); });
    each_k("lbvh_refit (BVH4)", 0xFFFFFFFFu, true, [&](std::vector<void *> *) { return refit(true); });

    // The device view of an engine (Engine::dev_scene) across failed updates: a one-quad scene, an environment map and the lookup tables,
    // then set_env_map, set_luts and set_material's emissive rebuild with their k-th allocation failing.  After every call each non-null
    // pointer of the view lies in a live block and the readiness checks agree with the view.
    {
        const std::set<void *> before_engine = g_live;
        setenv("B200PT_BVH_SAH", "0", 1);                          // the plain LBVH: the host tree passes need real boxes
        {
            Engine e(0);
            auto view_ok = [&](const char *what, long k) {
                const DevScene sc = e.dev_scene();
                const void *ptrs[] = { sc.verts, sc.indices, sc.meshes, sc.instances, sc.materials, sc.textures, sc.emissive, sc.env, sc.alias, sc.env_row_cos,
                                       sc.lut_reflect, sc.lut_refract_out, sc.lut_refract_in, sc.tri_slot, sc.tri_class, sc.nodes, sc.nodes4, sc.tris, sc.shade_tris,
                                       sc.em_tris, sc.em_tri_base, sc.volumes, sc.grids };
                bool ok = e.has_env() == (sc.env && sc.alias && sc.env_row_cos) && e.has_luts() == (sc.lut_reflect && sc.lut_refract_out && sc.lut_refract_in);
                for (const void *p : ptrs) ok = ok && (!p || live(p));
                expect(ok, what, k);
            };
            auto code = [](auto f) { try { f(); } catch (const CudaError &err) { return err.code; } return (int)B200PT_OK; };
            // call() with its k-th creation failing, for k = 1, 2, ... until it succeeds; check(k, ok, prev, created): the view before the
            // call and the blocks the call left behind
            auto each_failure = [&](const char *name, auto call, auto check) {
                const int failures0 = failures;
                for (long k = 1;; k++) {
                    const DevScene prev = e.dev_scene();
                    const long serial0 = g_serial;
                    arm(k, 0);
                    const bool ok = code(call) == B200PT_OK;
                    const bool injected = g_created >= k;
                    arm(0, 0);
                    std::set<const void *> created;
                    for (const auto &b : g_blocks) if (b.second.serial > serial0) created.insert(b.first);
                    expect(ok != injected, name, k);
                    view_ok(name, k);
                    check(k, ok, prev, created);
                    if (!injected) { printf("%s: %ld creations, %d failed\n", name, k - 1, failures - failures0); return; }
                }
            };

            HostScene s;                                           // one quad, one instance, one material that emits nothing
            HostMesh quad;
            quad.vertices.resize(4);
            for (int v = 0; v < 4; v++) { quad.vertices[v].Position[0] = (float)(v & 1); quad.vertices[v].Position[1] = (float)(v >> 1); }
            quad.indices = { 0, 1, 2, 2, 1, 3 };
            s.meshes.push_back(quad);
            b200pt_material m{}; m.BaseColor[0] = m.BaseColor[1] = m.BaseColor[2] = 0.5f;
            m.BaseColorTextureIndex = m.NormalTextureIndex = m.RoughnessTextureIndex = m.MetallicTextureIndex = m.EmissiveTextureIndex = 0;
            s.materials.push_back(m);
            HostTexture white; white.width = white.height = 1; white.channels = 4; white.data = { 255, 255, 255, 255 };
            s.textures.push_back(white);
            b200pt_instance in{}; for (int i = 0; i < 4; i++) in.Transform[i * 5] = 1.0f;
            s.instances.push_back(in);
            for (int i = 0; i < 16; i++) s.camera_view[i] = (i % 5 == 0) ? 1.0f : 0.0f;
            s.camera_aspect = 1.0f;
            std::vector<float> rgba(4 * 2 * 4, 1.0f);
            const size_t lut_n[3] = { 64 * 64 * 32, 128 * 128 * 32, 128 * 128 * 32 };
            std::vector<float> lut[3] = { std::vector<float>(lut_n[0], 0.5f), std::vector<float>(lut_n[1], 0.5f), std::vector<float>(lut_n[2], 0.5f) };
            arm(0, 1u);                                            // lbvh_build: every triangle one reference
            int r = code([&] { e.set_scene(std::move(s)); e.set_env_map(2, 2, rgba.data()); e.set_luts(lut[0].data(), lut[1].data(), lut[2].data()); });
            expect(r == B200PT_OK && e.has_scene() && e.has_env() && e.has_luts(), "engine set up", 0);
            view_ok("engine set up", 0);
            auto refuses = [&](long k, bool env) {                 // every launch that reads the map (env) or the tables refuses
                float out[64] = {}; const float dir[3] = { 0.0f, 0.0f, 1.0f }, pdf = 1.0f; const uint32_t depth = 1, u0 = 0; uint32_t survivors = 0;
                expect(code([&] { e.path_trace(1, 0); }) == B200PT_ERR_NO_SCENE && (!env || code([&] { e.miss_query(1, dir, &depth, &pdf, out); }) == B200PT_ERR_NO_SCENE) &&
                       code([&] { e.shade_query(false, 1, &u0, &u0, out, dir, dir, &pdf, &u0, nullptr, out); }) == B200PT_ERR_NO_SCENE &&
                       code([&] { e.bounce_query(1, out, 0, out, &survivors); }) == B200PT_ERR_NO_SCENE, "refused without the map or the tables", k);
            };

            each_failure("set_env_map", [&] { e.set_env_map(4, 2, rgba.data()); }, [&](long k, bool ok, const DevScene &, const std::set<const void *> &created) {
                const DevScene sc = e.dev_scene();
                if (ok) expect(e.has_env() && created == std::set<const void *>{ sc.env, sc.alias, sc.env_row_cos } && sc.envW == 4 && sc.envH == 2,
                               "set_env_map: the view holds the new map", k);
                else { expect(!e.has_env() && created.empty(), "failed set_env_map: no map, nothing of the call live", k); refuses(k, true); }
            });
            each_failure("set_luts", [&] { e.set_luts(lut[0].data(), lut[1].data(), lut[2].data()); }, [&](long k, bool ok, const DevScene &, const std::set<const void *> &created) {
                const DevScene sc = e.dev_scene();
                if (ok) expect(e.has_luts() && created == std::set<const void *>{ sc.lut_reflect, sc.lut_refract_out, sc.lut_refract_in }, "set_luts: the view holds the new tables", k);
                else { expect(!e.has_luts() && created.empty(), "failed set_luts: no tables, nothing of the call live", k); refuses(k, false); }
            });
            m.EmissiveColor[0] = 1.0f;                             // the quad becomes an emitter: two EmTri
            each_failure("set_material", [&] { e.set_material(0, m); }, [&](long k, bool ok, const DevScene &prev, const std::set<const void *> &created) {
                const DevScene sc = e.dev_scene();
                if (ok) expect(sc.n_emissive == 1 && created == std::set<const void *>{ sc.em_tris, sc.em_tri_base } && g_blocks.at((const char *)sc.em_tris).bytes == 2 * sizeof(EmTri),
                               "set_material: the view holds the new emissive tables", k);
                else expect(sc.n_emissive == 0 && sc.em_tris == prev.em_tris && sc.em_tri_base == prev.em_tri_base && created.empty(),
                            "failed set_material: the previous emissive tables", k);
            });
        }
        unsetenv("B200PT_BVH_SAH");
        expect(g_live == before_engine, "engine destroyed: nothing live", 0);
    }
    if (failures) { printf("%d failures\n", failures); return 1; }
    puts("ok");
    return 0;
}
