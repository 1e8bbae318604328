// animation.cpp -- a pose of a loaded glTF scene on the host: channels sampled at time t as glTF 2.0 Appendix C defines it, node world
// matrices, joint matrices and morph weights.  No CUDA in here: the pose query hook runs without a GPU, and Engine::pose hands the result
// to pose_kernels.cu.
//
// Exactness: channels are sampled in double and rounded to float; node world matrices then use the loader's own float arithmetic (node_local,
// m4_mul, the flip), so a node no channel touches keeps, bit for bit, the instance transform it had at load.
#include "host_api.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace b200pt {

static void bad(const std::string &what) { throw CudaError{ B200PT_ERR_WRONG_ARGUMENTS, what }; }

uint32_t animation_range(const AnimClip &c, float *t0, float *t1) {
    bool any = false; float lo = 0.0f, hi = 0.0f;
    for (const AnimChannel &ch : c.channels) {
        const AnimSampler &s = c.samplers[ch.sampler];
        if (s.input.empty()) continue;
        if (!any || s.input.front() < lo) lo = s.input.front();
        if (!any || s.input.back() > hi) hi = s.input.back();
        any = true;
    }
    *t0 = lo; *t1 = hi;
    return (uint32_t)c.channels.size();
}

// The deformable meshes: those an instance deforms through a skin or morph targets.  A mesh its instances would deform differently (different
// skins, or one skinned and one not) is deformable and carries the error.  Also: joint indices against the skin, the node graph a forest.
void finalize_animation(HostAnimation &a, const HostScene &sc) {
    const size_t nm = sc.meshes.size();
    a.prim_skin.assign(nm, -1);
    std::vector<uint8_t> seen(nm, 0), conflict(nm, 0);
    for (size_t i = 0; i < sc.instances.size() && i < a.instance_node.size(); i++) {
        const uint32_t p = sc.instances[i].MeshIndex; const int skin = a.nodes[a.instance_node[i]].skin;
        if (!seen[p]) { seen[p] = 1; a.prim_skin[p] = skin; }
        else if (a.prim_skin[p] != skin) conflict[p] = 1;
    }
    a.deformable.clear();
    for (size_t p = 0; p < nm; p++) {
        AnimPrim &ap = a.prims[p];
        if (!seen[p] || !(ap.targets || a.prim_skin[p] >= 0 || conflict[p])) continue;
        a.deformable.push_back((int)p);
        if (conflict[p] && ap.err.empty()) ap.err = "mesh " + std::to_string(p) + " is deformed two ways by the nodes that instance it (different skins, or skinned and not)";
        const int s = a.prim_skin[p];
        if (s >= 0 && ap.err.empty()) {
            if (!ap.sets) ap.err = "skinned mesh " + std::to_string(p) + " has no JOINTS_0 / WEIGHTS_0";
            for (uint32_t j : ap.joints) if (j >= a.skins[s].joints.size()) { ap.err = "mesh " + std::to_string(p) + ": joint index out of the skin's range"; break; }
        }
    }
    // every node has at most one parent, no root is a child, and there is no cycle (the parent walks of evaluate_pose end)
    std::vector<int> parent(a.nodes.size(), -1);
    for (size_t n = 0; n < a.nodes.size(); n++)
        for (int c : a.nodes[n].children) {
            if (parent[c] >= 0 && a.err.empty()) a.err = "node " + std::to_string(c) + " has two parents";
            parent[c] = (int)n;
        }
    for (int r : a.roots) if (r >= 0 && (size_t)r < parent.size() && parent[r] >= 0 && a.err.empty()) a.err = "root node " + std::to_string(r) + " is a child";
    for (size_t n = 0; n < a.nodes.size() && a.err.empty(); n++) {
        size_t steps = 0;
        for (int k = (int)n; k >= 0; k = parent[k]) if (++steps > a.nodes.size()) { a.err = "the node graph has a cycle"; break; }
    }
}

// glTF 2.0 Appendix C: one channel's value at t (clamped to the keys), in double
static void sample(const AnimSampler &s, double t, bool rotation, double *v) {
    const uint32_t n = s.comps; const size_t K = s.input.size();
    const bool cubic = s.interp == INTERP_CUBIC;
    auto val = [&](size_t k) { return &s.output[(cubic ? 3 * k + 1 : k) * n]; };
    if (K == 1 || t <= s.input[0]) { for (uint32_t c = 0; c < n; c++) v[c] = val(0)[c]; return; }
    if (t >= s.input[K - 1]) { for (uint32_t c = 0; c < n; c++) v[c] = val(K - 1)[c]; return; }
    const size_t k = (size_t)(std::upper_bound(s.input.begin(), s.input.end(), (float)t, [](float a, float b) { return a < b; }) - s.input.begin()) - 1;
    const size_t kk = std::min(k, K - 2);
    const double ta = s.input[kk], tb = s.input[kk + 1], td = tb - ta, u = std::min(std::max((t - ta) / td, 0.0), 1.0);
    const float *a = val(kk), *b = val(kk + 1);
    if (s.interp == INTERP_STEP) { for (uint32_t c = 0; c < n; c++) v[c] = a[c]; return; }
    if (s.interp == INTERP_LINEAR) {
        if (!rotation) { for (uint32_t c = 0; c < n; c++) v[c] = (1.0 - u) * a[c] + u * b[c]; return; }
        double d = 0.0; for (int c = 0; c < 4; c++) d += (double)a[c] * b[c];
        const double sg = d < 0.0 ? -1.0 : 1.0, ad = std::fabs(d);
        if (ad > 1.0 - 1e-9) { for (int c = 0; c < 4; c++) v[c] = (1.0 - u) * a[c] + sg * u * b[c]; return; }   // tiny angle: linear
        const double ang = std::acos(ad), sa = std::sin(ang), wa = std::sin(ang * (1.0 - u)) / sa, wb = sg * std::sin(ang * u) / sa;
        for (int c = 0; c < 4; c++) v[c] = wa * a[c] + wb * b[c];
        return;
    }
    // CUBICSPLINE: [in-tangent, value, out-tangent] per key, tangents scaled by the key interval
    const float *bk = &s.output[(3 * kk + 2) * n], *ak1 = &s.output[(3 * (kk + 1)) * n];
    const double u2 = u * u, u3 = u2 * u;
    const double h00 = 2 * u3 - 3 * u2 + 1, h10 = td * (u3 - 2 * u2 + u), h01 = -2 * u3 + 3 * u2, h11 = td * (u3 - u2);
    for (uint32_t c = 0; c < n; c++) v[c] = h00 * a[c] + h10 * bk[c] + h01 * b[c] + h11 * ak1[c];
    if (rotation) {
        double l = 0.0; for (int c = 0; c < 4; c++) l += v[c] * v[c];
        l = std::sqrt(l); if (l > 0.0) for (int c = 0; c < 4; c++) v[c] /= l;
    }
}

void evaluate_pose(const HostAnimation &a, const HostScene &sc, int animation, float t, HostPose &out) {
    if (!a.err.empty()) bad(a.err);
    if (animation >= (int)a.clips.size()) bad("animation index out of range");
    const size_t nn = a.nodes.size();
    std::vector<NodeTRS> trs(nn);
    out.weights.assign(nn, {});
    for (size_t i = 0; i < nn; i++) {
        trs[i] = a.nodes[i].trs;
        const int m = a.nodes[i].mesh;
        if (m < 0 || !a.mesh_targets[m]) continue;
        out.weights[i] = a.nodes[i].has_weights ? a.nodes[i].weights : !a.mesh_weights[m].empty() ? a.mesh_weights[m] : std::vector<float>(a.mesh_targets[m], 0.0f);
    }
    if (animation >= 0) {
        const AnimClip &c = a.clips[animation];
        if (!c.err.empty()) bad("animation " + std::to_string(animation) + ": " + c.err);
        double v[256];
        for (const AnimChannel &ch : c.channels) {
            const AnimSampler &s = c.samplers[ch.sampler];
            sample(s, (double)t, ch.path == PATH_R, v);
            float *dst = ch.path == PATH_T ? trs[ch.node].t : ch.path == PATH_R ? trs[ch.node].r : ch.path == PATH_S ? trs[ch.node].s : out.weights[ch.node].data();
            for (uint32_t k = 0; k < s.comps; k++) dst[k] = (float)v[k];
        }
    }
    // world matrices: parent world x local, roots from the identity, as the loader's depth-first walk multiplies them
    std::vector<int> parent(nn, -1);
    for (size_t n = 0; n < nn; n++) for (int c : a.nodes[n].children) parent[c] = (int)n;
    out.world.assign(nn, m4_identity());
    std::vector<uint8_t> done(nn, 0); std::vector<int> chain;
    for (size_t n = 0; n < nn; n++) {
        chain.clear();
        for (int k = (int)n; k >= 0 && !done[k]; k = parent[k]) chain.push_back(k);
        for (size_t i = chain.size(); i-- > 0;) {
            const int k = chain[i];
            out.world[k] = m4_mul(parent[k] >= 0 ? out.world[parent[k]] : m4_identity(), node_local(trs[k]));
            done[k] = 1;
        }
    }
    // instances: flip x world, except skinned meshes, whose vertices are posed in glTF world space (glTF 2.0 3.7.3.3)
    M4 flip = m4_identity(); flip.m[1][1] = -1.0f;
    out.instances = sc.instances;
    for (size_t i = 0; i < out.instances.size(); i++) {
        const uint32_t p = out.instances[i].MeshIndex;
        if (a.prim_skin[p] >= 0) m4_to_colmajor(flip, out.instances[i].Transform);
        else m4_to_colmajor(m4_mul(flip, out.world[a.instance_node[i]]), out.instances[i].Transform);
    }
    // per deformable mesh: the joint palette world(joint) x inverseBind and the morph weights, checked against every instance of the mesh
    out.palette.clear(); out.palette_base.assign(1, 0); out.morph.clear(); out.morph_base.assign(1, 0);
    for (int p : a.deformable) {
        const AnimPrim &ap = a.prims[p];
        if (!ap.err.empty()) bad(ap.err);
        const int s = a.prim_skin[p];
        if (s >= 0) {
            const AnimSkin &S = a.skins[s];
            if (!S.err.empty()) bad(S.err);
            for (size_t j = 0; j < S.joints.size(); j++) {
                const M4 J = m4_mul(out.world[S.joints[j]], S.inverse_bind[j]);
                for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++) out.palette.push_back(J.m[r][c]);
            }
        }
        out.palette_base.push_back((uint32_t)(out.palette.size() / 12));
        if (ap.targets) {
            const std::vector<float> *w = nullptr;
            for (size_t i = 0; i < sc.instances.size(); i++) {
                if (sc.instances[i].MeshIndex != (uint32_t)p) continue;
                const std::vector<float> &wi = out.weights[a.instance_node[i]];
                if (!w) w = &wi;
                else if (wi.size() != w->size() || (!wi.empty() && memcmp(wi.data(), w->data(), wi.size() * sizeof(float))))
                    bad("mesh " + std::to_string(p) + " is deformed two ways: the nodes that instance it have different morph weights");
            }
            for (uint32_t k = 0; k < ap.targets; k++) {
                const float x = (*w)[k];
                if (!std::isfinite(x)) bad("morph weight is not finite");
                out.morph.push_back(x);
            }
        }
        out.morph_base.push_back((uint32_t)out.morph.size());
    }
    for (const M4 &w : out.world) for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) if (!std::isfinite(w.m[r][c])) bad("a node's world matrix is not finite");
    for (float x : out.palette) if (!std::isfinite(x)) bad("a joint matrix is not finite");
}

} // namespace b200pt
