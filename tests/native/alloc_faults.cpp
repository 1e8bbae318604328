// Host-only check that the host runtime leaves no CUDA resource behind on any error path.  The runtime calls that create, copy and
// release are replaced by shims defined in THIS file (the executable's own symbols win over libcudart's, as in refine_plumbing.cpp):
// device and pinned memory are zeroed host blocks, events and streams are host blocks as well, every live one is tracked, kernel
// launches do nothing, and a device-to-host copy fills its destination with a chosen word (what the builders read back).  For every k:
//   * Engine (b200pt_create): the k-th creation of a stream, event or block fails; nothing is live after the error, nor after
//     b200pt_destroy of an engine whose creation succeeded;
//   * lbvh_build, ploc_build, lbvh_ploc_rebuild, bvh4_collapse_device, lbvh_build_wide_device: the k-th cudaMalloc fails; a failing
//     call leaves nothing live, a successful call exactly its outputs;
//   * lbvh_build of a scene whose split counts add up to 2^28 references returns an error and leaves nothing live.
// Built and run by tests/test_resource_ownership.py: nvcc --cudart shared ... tests/native/alloc_faults.cpp <every object of build/> -lz
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <vector>
#include <cuda_runtime.h>
#include "kernels.h"
#include "b200pt.h"
using namespace b200pt;

static long g_fail_at = 0, g_created = 0;      // creations since the last arm(); the g_fail_at-th fails (0: none)
static std::set<void *> g_live;
static uint32_t g_readback = 0;

static void arm(long k, uint32_t readback) { g_fail_at = k; g_created = 0; g_readback = readback; }
static cudaError_t create(void **p, size_t bytes) {
    *p = nullptr;
    if (++g_created == g_fail_at) return cudaErrorMemoryAllocation;
    *p = calloc(1, bytes ? bytes : 1);
    g_live.insert(*p);
    return cudaSuccess;
}
static cudaError_t release(void *p) {
    if (!p) return cudaSuccess;
    if (!g_live.erase(p)) { printf("FAIL: release of a handle that is not live\n"); exit(1); }
    free(p);
    return cudaSuccess;
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
        LbvhResult res{}; DevPtr<float> ref_box;
        const int r = lbvh_build(verts.data(), idx.data(), &mesh, &inst, &inst, &mesh, 1, n_tris, &res, nullptr, true, &ref_box);
        if (r == 0) { *outs = { res.shade, res.tri_slot, res.nodes, ref_box.release() }; free(res.h_ref_box); }
        else lbvh_free(&res);
        return r;
    };
    each_k("lbvh_build", 1u, true, [&](std::vector<void *> *o) { return build(nt, o); });
    each_k("lbvh_build (2^28 references)", 1u << 20, false, [&](std::vector<void *> *o) {
        const int r = build(256, o);
        if (r == 0) { printf("FAIL: 2^28 references accepted\n"); failures++; }
        return r;
    });

    // the device tree builder and collapse on host arrays: one clustering step (cluster count read back as 1), one BVH4 level (0)
    std::vector<float> boxes((size_t)nt * 6, 0.0f); std::vector<BvhNode> nodes(nt - 1), nodes2(nt - 1); std::vector<uint32_t> perm(nt), slot(nt);
    std::vector<BvhTri> tris(nt); std::vector<Bvh4Node> nodes4(nt - 1);
    each_k("ploc_build", 1u, true, [&](std::vector<void *> *) {
        uint32_t n_out = 0; int depth = 0; uint32_t h_small[4];
        return ploc_build(boxes.data(), nt, nodes.data(), perm.data(), &n_out, &depth, h_small, nullptr);
    });
    each_k("lbvh_ploc_rebuild", 1u, true, [&](std::vector<void *> *) {
        LbvhResult res{}; res.nodes = nodes.data(); res.tris = tris.data(); res.tri_slot = slot.data(); res.n_nodes = nt - 1; res.n_tris = res.n_prims = nt;
        res.max_depth = 10;
        const long k = g_fail_at; arm(0, 1u);                     // the reference boxes come from the caller, beside the count
        DevPtr<float> ref_box; alloc(ref_box, (size_t)nt * 6 * sizeof(float)); arm(k, 1u);
        uint32_t h_small[4];
        return lbvh_ploc_rebuild(&res, std::move(ref_box), h_small, nullptr);
    });
    each_k("bvh4_collapse_device", 0u, true, [&](std::vector<void *> *) {
        uint32_t n4 = 0, h_total[4]; int d4 = 0;
        return bvh4_collapse_device(nodes2.data(), nt - 1, 0, nodes4.data(), &n4, &d4, h_total, nullptr);
    });
    each_k("lbvh_build_wide_device", 0u, true, [&](std::vector<void *> *o) {
        LbvhResult res{}; res.nodes = nodes2.data(); res.n_nodes = nt - 1;
        uint32_t h_small[4];
        const int r = lbvh_build_wide_device(&res, h_small, nullptr);
        *o = { res.nodes4 };
        return r;
    });
    if (failures) { printf("%d failures\n", failures); return 1; }
    puts("ok");
    return 0;
}
