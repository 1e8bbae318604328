// Host-only check of lbvh_refine_sah's plumbing (csrc/lbvh.cu): the CUDA copies are replaced by memcpy shims defined in THIS file
// (the executable's own symbols win over libcudart's), and cudaFree by a no-op because the result's owners wrap host vectors, so the
// function runs on host arrays without a GPU.  For every mode 1..5:
//   * every ray finds the same closest triangle id and distance in the refined structure as by brute force over all triangles,
//   * tri_slot[gid] points at a slot that holds triangle gid, root == 0, max_depth == the depth of the emitted tree.
// Build and run by hand (or through tests/test_host_api.py::test_refine_sah_plumbing_with_caller_reference_boxes, which does exactly this):
//   nvcc -std=c++17 -O1 -gencode arch=compute_90a,code=sm_90a -Ivulkan-path-tracer_b200/csrc -Iinclude tests/native/refine_plumbing.cpp vulkan-path-tracer_b200/build/lbvh.o -o /tmp/refine_plumbing
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>
#include <random>
#include <algorithm>
#include <cuda_runtime.h>
#include "kernels.h"
using namespace b200pt;

extern "C" {
cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(dst, src, n); return cudaSuccess; }
cudaError_t cudaMemcpy(void *dst, const void *src, size_t n, cudaMemcpyKind) { memcpy(dst, src, n); return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaFree(void *) { return cudaSuccess; }
}

struct Hit { float t; uint32_t gid; };
static bool tri_hit(const BvhTri &T, const float o[3], const float d[3], float &t) {
    const double e1[3] = { T.b.x, T.b.y, T.b.z }, e2[3] = { T.c.x, T.c.y, T.c.z }, a[3] = { T.a.x, T.a.y, T.a.z };
    const double p[3] = { d[1] * e2[2] - d[2] * e2[1], d[2] * e2[0] - d[0] * e2[2], d[0] * e2[1] - d[1] * e2[0] };
    const double det = e1[0] * p[0] + e1[1] * p[1] + e1[2] * p[2];
    if (fabs(det) < 1e-30) return false;
    const double s[3] = { o[0] - a[0], o[1] - a[1], o[2] - a[2] };
    const double u = (s[0] * p[0] + s[1] * p[1] + s[2] * p[2]) / det;
    const double q[3] = { s[1] * e1[2] - s[2] * e1[1], s[2] * e1[0] - s[0] * e1[2], s[0] * e1[1] - s[1] * e1[0] };
    const double v = (d[0] * q[0] + d[1] * q[1] + d[2] * q[2]) / det, tt = (e2[0] * q[0] + e2[1] * q[1] + e2[2] * q[2]) / det;
    if (u < 0 || v < 0 || u + v > 1 || tt <= 1e-6) return false;
    t = (float)tt; return true;
}
static uint32_t gid_of(const BvhTri &T) { uint32_t g; memcpy(&g, &T.a.w, 4); return g; }
static Hit walk(const std::vector<BvhNode> &nodes, int32_t root, const std::vector<BvhTri> &tris, const float o[3], const float d[3], int *max_stack) {
    Hit h{ 3.0e38f, 0xFFFFFFFFu };
    std::vector<int32_t> st{ root };
    while (!st.empty()) {
        if ((int)st.size() > *max_stack) *max_stack = (int)st.size();
        const int32_t c = st.back(); st.pop_back();
        if (c < 0) {
            const uint32_t r = (uint32_t)~c, first = r >> 2, cnt = (r & 3u) + 1u;
            for (uint32_t k = 0; k < cnt; k++) { float t; if (tri_hit(tris[first + k], o, d, t)) { const uint32_t g = gid_of(tris[first + k]); if (t < h.t || (t == h.t && g < h.gid)) { h.t = t; h.gid = g; } } }
            continue;
        }
        const BvhNode &N = nodes[c];
        for (int k = 0; k < 2; k++) {
            const float *lo = k ? N.lo1 : N.lo0, *hi = k ? N.hi1 : N.hi0;
            float tn = 0.0f, tf = h.t;
            for (int a = 0; a < 3; a++) { const float inv = 1.0f / d[a]; float t0 = (lo[a] - o[a]) * inv, t1 = (hi[a] - o[a]) * inv; if (t0 > t1) std::swap(t0, t1); tn = fmaxf(tn, t0); tf = fminf(tf, t1); }
            if (tn <= tf) st.push_back(k ? N.c1 : N.c0);
        }
    }
    return h;
}
static int depth_of(const std::vector<BvhNode> &nodes, int32_t n) { if (n < 0) return 0; return 1 + std::max(depth_of(nodes, nodes[n].c0), depth_of(nodes, nodes[n].c1)); }

int main() {
    std::mt19937 rng(11); std::uniform_real_distribution<float> U(0.f, 1.f);
    for (int scene = 0; scene < 6; scene++) {
        const uint32_t n_prims = scene < 2 ? 11 : 3000 + 500 * scene;
        // triangles; every 7th gets two reference slots (as the split clipping of fat triangles does)
        std::vector<BvhTri> base; std::vector<float> boxes;
        for (uint32_t g = 0; g < n_prims; g++) {
            BvhTri T; const float c[3] = { U(rng) * 4 - 2, U(rng) * 4 - 2, U(rng) * 4 - 2 };
            float v[3][3]; for (auto &x : v) for (int a = 0; a < 3; a++) x[a] = c[a] + 0.3f * (U(rng) - 0.5f);
            T.a = make_float4(v[0][0], v[0][1], v[0][2], 0.f); memcpy(&T.a.w, &g, 4);
            T.b = make_float4(v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2], 0.f);
            T.c = make_float4(v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2], 0.f);
            float lo[3], hi[3]; for (int a = 0; a < 3; a++) { lo[a] = fminf(v[0][a], fminf(v[1][a], v[2][a])); hi[a] = fmaxf(v[0][a], fmaxf(v[1][a], v[2][a])); }
            const int refs = (g % 7 == 3) ? 2 : 1;
            for (int r = 0; r < refs; r++) {
                base.push_back(T);
                float l2[3] = { lo[0], lo[1], lo[2] }, h2[3] = { hi[0], hi[1], hi[2] };
                if (refs == 2) { const float mid = 0.5f * (lo[0] + hi[0]); if (r == 0) h2[0] = mid; else l2[0] = mid; }
                for (int a = 0; a < 3; a++) boxes.push_back(l2[a]); for (int a = 0; a < 3; a++) boxes.push_back(h2[a]);
            }
        }
        // note: a split reference only bounds part of its triangle; a ray through the other part reaches it through the sibling reference
        const uint32_t n = (uint32_t)base.size();
        // stand-in for the GPU LBVH: slots sorted along x only, median splits in index order, leaves of <= 4 consecutive slots, padded boxes
        std::vector<uint32_t> perm(n); for (uint32_t i = 0; i < n; i++) perm[i] = i;
        std::sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return boxes[(size_t)a * 6] + boxes[(size_t)a * 6 + 3] < boxes[(size_t)b * 6] + boxes[(size_t)b * 6 + 3]; });
        std::vector<BvhTri> tris0(n); std::vector<float> boxes0((size_t)n * 6); std::vector<uint32_t> slot0(n_prims);
        for (uint32_t i = 0; i < n; i++) { tris0[i] = base[perm[i]]; memcpy(&boxes0[(size_t)i * 6], &boxes[(size_t)perm[i] * 6], 24); slot0[gid_of(tris0[i])] = i; }
        std::vector<BvhNode> init; int d0 = 0;
        struct Rg { uint32_t b, e; int32_t parent; int side; int dep; };
        std::vector<Rg> todo{ { 0, n, -1, 0, 1 } };
        auto bounds = [&](uint32_t b, uint32_t e, float lo[3], float hi[3]) {
            for (int a = 0; a < 3; a++) { lo[a] = 3e38f; hi[a] = -3e38f; }
            for (uint32_t i = b; i < e; i++) for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], boxes0[(size_t)i * 6 + a]); hi[a] = fmaxf(hi[a], boxes0[(size_t)i * 6 + 3 + a]); }
            for (int a = 0; a < 3; a++) { lo[a] -= 1e-5f; hi[a] += 1e-5f; }
        };
        while (!todo.empty()) {
            const Rg g = todo.back(); todo.pop_back();
            const int32_t me = (int32_t)init.size(); init.push_back(BvhNode{});
            if (g.parent >= 0) (g.side ? init[g.parent].c1 : init[g.parent].c0) = me;
            if (g.dep > d0) d0 = g.dep;
            const uint32_t mid = g.b + (g.e - g.b) / 2;
            bounds(g.b, mid, init[me].lo0, init[me].hi0); bounds(mid, g.e, init[me].lo1, init[me].hi1);
            if (mid - g.b <= 4) init[me].c0 = ~(int32_t)((g.b << 2) | (mid - g.b - 1)); else todo.push_back({ g.b, mid, me, 0, g.dep + 1 });
            if (g.e - mid <= 4) init[me].c1 = ~(int32_t)((mid << 2) | (g.e - mid - 1)); else todo.push_back({ mid, g.e, me, 1, g.dep + 1 });
        }
        const uint32_t n0 = (uint32_t)init.size();
        // shuffle the initial inner nodes so that the root is not node 0 and children do not follow parents (as in the Karras layout)
        std::vector<uint32_t> order(n0); for (uint32_t i = 0; i < n0; i++) order[i] = i;
        std::shuffle(order.begin(), order.end(), rng);
        std::vector<BvhNode> shuf(n - 1);
        for (uint32_t i = 0; i < n0; i++) { BvhNode N = init[i]; if (N.c0 >= 0) N.c0 = (int32_t)order[N.c0]; if (N.c1 >= 0) N.c1 = (int32_t)order[N.c1]; shuf[order[i]] = N; }
        const int32_t root0 = (int32_t)order[0];
        // rays + brute force
        const int R = 300; std::vector<float> O(R * 3), D(R * 3); std::vector<Hit> truth(R);
        for (int r = 0; r < R; r++) {
            const BvhTri &T = base[rng() % n]; float tgt[3] = { T.a.x + 0.3f * (T.b.x + T.c.x), T.a.y + 0.3f * (T.b.y + T.c.y), T.a.z + 0.3f * (T.b.z + T.c.z) };
            float len = 0; for (int a = 0; a < 3; a++) { O[r * 3 + a] = U(rng) * 6 - 3; D[r * 3 + a] = tgt[a] - O[r * 3 + a]; len += D[r * 3 + a] * D[r * 3 + a]; }
            len = sqrtf(len); for (int a = 0; a < 3; a++) { D[r * 3 + a] /= len; if (fabsf(D[r * 3 + a]) < 1e-6f) D[r * 3 + a] = 1e-6f; }
            Hit h{ 3.0e38f, 0xFFFFFFFFu };
            for (uint32_t i = 0; i < n; i++) { float t; if (tri_hit(base[i], &O[r * 3], &D[r * 3], t)) { const uint32_t g = gid_of(base[i]); if (t < h.t || (t == h.t && g < h.gid)) { h.t = t; h.gid = g; } } }
            truth[r] = h;
        }
        for (int mode = 0; mode <= 5; mode++) {
            LbvhResult res{}; std::vector<BvhNode> nodes = shuf; std::vector<BvhTri> tris = tris0; std::vector<uint32_t> slot = slot0; std::vector<float> rb = boxes0;
            res.nodes.reset(nodes.data()); res.tris = tris.data(); res.tri_slot.reset(slot.data()); res.n_nodes = n - 1; res.n_tris = n; res.root = root0; res.max_depth = d0;
            res.n_prims = n_prims;
            const float *ref_box = (mode == 2 || mode == 3) ? rb.data() : nullptr;
            double sah[2] = { 0, 0 };
            if (mode && lbvh_refine_sah(&res, ref_box, nullptr, sah, mode) != 0) { printf("mode %d failed\n", mode); return 1; }
            const bool kept = mode && res.root == root0 && sah[1] == sah[0];   // the pass found nothing cheaper and left the structure alone
            if (mode && !kept && (res.root != 0 || !(sah[1] < sah[0]))) { printf("scene %d mode %d: root %d cost %g -> %g\n", scene, mode, res.root, sah[0], sah[1]); return 1; }
            if (res.max_depth != depth_of(nodes, res.root)) { printf("scene %d mode %d: max_depth %d != %d\n", scene, mode, res.max_depth, depth_of(nodes, res.root)); return 1; }
            for (uint32_t g = 0; g < n_prims; g++) if (slot[g] >= n || gid_of(tris[slot[g]]) != g) { printf("scene %d mode %d: tri_slot[%u] broken\n", scene, mode, g); return 1; }
            int max_stack = 0, hits = 0;
            for (int r = 0; r < R; r++) {
                const Hit h = walk(nodes, res.root, tris, &O[r * 3], &D[r * 3], &max_stack);
                if (h.gid != truth[r].gid || h.t != truth[r].t) { printf("scene %d mode %d ray %d: tree (%u, %g) vs brute force (%u, %g)\n", scene, mode, r, h.gid, h.t, truth[r].gid, truth[r].t); return 1; }
                hits += h.gid != 0xFFFFFFFFu;
            }
            if (hits < R / 2) { printf("scene %d: only %d hits\n", scene, hits); return 1; }
            if (max_stack > res.max_depth + 2) { printf("scene %d mode %d: stack %d > depth %d + 2\n", scene, mode, max_stack, res.max_depth); return 1; }
            printf("scene %d (%u prims, %u slots) mode %d: ok, cost %.2f -> %.2f, depth %d, stack %d\n", scene, n_prims, n, mode, sah[0], sah[1], res.max_depth, max_stack);
        }
    }
    puts("ok");
    return 0;
}
