// Sanitizer harness for the host restatement of the GPU tree builder (bvh2_ploc_build_host, csrc/lbvh.cu), beside fuzz_bvh_passes.cpp:
// random reference sets in Morton-like order (scattered, coplanar, identical, overlapping, nested scales, huge and degenerate extents), each
// built, then the result collapsed to a BVH4 and refined by re-insertion, which must accept it as a tree.
// Not part of the pytest run; build and run by hand:
//   S=vulkan-path-tracer_b200/csrc; F="-Xcompiler -fsanitize=address -Xcompiler -fsanitize=undefined"
//   nvcc -std=c++17 -O1 -g -gencode arch=compute_90a,code=sm_90a $F -I$S -Iinclude -c $S/lbvh.cu -o /tmp/lbvh_san.o
//   nvcc -std=c++17 -O1 -g -gencode arch=compute_90a,code=sm_90a $F -I$S -Iinclude tests/native/fuzz_ploc_build.cpp /tmp/lbvh_san.o -o /tmp/fuzz_ploc -lcudart
//   ASAN_OPTIONS=protect_shadow_gap=0:detect_leaks=0 /tmp/fuzz_ploc        (no GPU needed: only host functions are called)
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>
#include <cuda_runtime.h>
#include "kernels.h"
using namespace b200pt;
int main() {
    std::mt19937 rng(11);
    std::uniform_real_distribution<float> U(0.f, 1.f);
    for (int iter = 0; iter < 300; iter++) {
        const int mode = iter % 6;
        // all-equal distances (identical boxes, infinite areas) merge one pair per clustering step, so as many steps as references: keep
        // those sets small
        const uint32_t n = 5 + rng() % (iter < 250 || mode == 2 || mode == 5 ? 400 : (iter < 290 ? 20000 : 150000));
        std::vector<float> rb((size_t)n * 6);
        for (uint32_t i = 0; i < n; i++) {
            float c[3] = { U(rng), U(rng), U(rng) }, e = 0.01f * U(rng);
            if (mode == 1) c[0] = 0.5f;                                        // coplanar centroids
            if (mode == 2) { c[0] = c[1] = c[2] = 0.25f; }                     // all identical
            if (mode == 3) e = 0.5f * U(rng);                                  // overlapping
            if (mode == 4) { const float s = powf(0.55f, (float)(i % 40)); for (float &x : c) x = (x * 2 - 1) * s; e = 0.05f * s; }    // nested scales (not down to zero areas)
            if (mode == 5) { e = (i % 7 == 0) ? 0.0f : 1e30f * U(rng); }       // degenerate and huge extents (inf areas)
            for (int a = 0; a < 3; a++) { rb[i * 6 + a] = c[a] - e; rb[i * 6 + 3 + a] = c[a] + e; }
        }
        // Morton-like order: sort by the x centroid bucket, then y, then z (the builder only needs some locality)
        std::vector<uint32_t> order(n); for (uint32_t i = 0; i < n; i++) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return rb[x * 6] + rb[x * 6 + 3] < rb[y * 6] + rb[y * 6 + 3]; });
        std::vector<float> sorted((size_t)n * 6);
        for (uint32_t i = 0; i < n; i++) std::copy(&rb[(size_t)order[i] * 6], &rb[(size_t)order[i] * 6 + 6], &sorted[(size_t)i * 6]);
        std::vector<BvhNode> nodes(n), out(n); std::vector<uint32_t> perm(n); int d = 0; double c = 0, s[2];
        const uint32_t m = bvh2_ploc_build_host(sorted.data(), n, nodes.data(), perm.data(), &d, &c);
        if (m == 0 || m > n - 1) { printf("build failed n=%u mode=%d\n", n, mode); return 1; }
        std::vector<uint8_t> seen(n, 0);
        for (uint32_t i = 0; i < n; i++) { if (perm[i] >= n || seen[perm[i]]) { printf("perm is not a permutation\n"); return 1; } seen[perm[i]] = 1; }
        std::vector<Bvh4Node> n4(m); int d4 = 0;
        if (bvh4_collapse_host(nodes.data(), m, 0, n4.data(), &d4) == 0) { printf("collapse failed\n"); return 1; }
        if (m >= 2 && bvh2_reinsert_host(nodes.data(), m, 0, out.data(), 1, 0.2f, &d, s) != m) { printf("not a tree\n"); return 1; }
    }
    puts("ok");
    return 0;
}
