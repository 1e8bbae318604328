// scene_loader.cpp -- glTF 2.0 scene loader reproducing the SceneAsset the reference's PathTracer consumes.
//
// Reference behaviour kept (VulkanHelper/Source/Utility/AssetImporterImpl.cpp, PathTracer/PathTracer.cpp):
//   * vertex {Position, normalize(Normal), TexCoord} 32 B, u32 indices          AssetImporterImpl.cpp:121-218
//   * instance Transform = diag(1,-1,1,1) * nodeWorld, depth-first node order    :220-262
//   * material keys + defaults (emissive * strength, metallic default 1, ior 1.5,
//     KHR_materials_{ior,transmission,specular,anisotropy,emissive_strength})    :353-455
//   * roughness AND metallic textures both = the metallicRoughness image, R channel only (PathTracer.cpp:826-836, Q8)
//   * texture table order + 1x1 defaults white / (128,128,255)                   PathTracer.cpp:228-408,1557-1621
//   * camera ViewMatrix = inverse(flipY * nodeWorld * local(right,-up,-lookAt))  AssetImporterImpl.cpp:547-642
// assimp (v6.0.2, network dependency, not vendored) is replaced by a direct glTF reader; its mesh merging
// (OptimizeMeshes/OptimizeGraph/JoinIdenticalVertices) only re-partitions geometry and is not reproduced.
#include "host_api.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <map>

namespace b200pt {

// ------------------------------------------------------------------------------------------------ minimal JSON
namespace {
struct JVal {
    enum T { Null, Bool, Num, Str, Arr, Obj } t = Null;
    bool b = false; double n = 0.0; std::string s;
    std::vector<JVal> a; std::vector<std::pair<std::string, JVal>> o;
    const JVal *get(const char *k) const { if (t != Obj) return nullptr; for (auto &kv : o) if (kv.first == k) return &kv.second; return nullptr; }
    bool has(const char *k) const { return get(k) != nullptr; }
    double num(const char *k, double def) const { const JVal *v = get(k); return (v && v->t == Num) ? v->n : def; }
    size_t size() const { return t == Arr ? a.size() : 0; }
    const JVal &operator[](size_t i) const { return a[i]; }
};
struct JParser {
    const char *p, *e; std::string err;
    void ws() { while (p < e && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) p++; }
    bool lit(const char *s) { size_t n = strlen(s); if ((size_t)(e - p) >= n && !strncmp(p, s, n)) { p += n; return true; } return false; }
    bool str(std::string &out) {
        if (p >= e || *p != '"') return false;
        p++;
        while (p < e && *p != '"') {
            if (*p == '\\' && p + 1 < e) {
                p++;
                switch (*p) {
                case 'n': out.push_back('\n'); break; case 't': out.push_back('\t'); break; case 'r': out.push_back('\r'); break;
                case 'b': out.push_back('\b'); break; case 'f': out.push_back('\f'); break;
                case 'u': { if (p + 4 < e) { unsigned cp = (unsigned)strtoul(std::string(p + 1, p + 5).c_str(), nullptr, 16); p += 4;
                            if (cp < 0x80) out.push_back((char)cp); else if (cp < 0x800) { out.push_back((char)(0xC0 | (cp >> 6))); out.push_back((char)(0x80 | (cp & 63))); }
                            else { out.push_back((char)(0xE0 | (cp >> 12))); out.push_back((char)(0x80 | ((cp >> 6) & 63))); out.push_back((char)(0x80 | (cp & 63))); } } } break;
                default: out.push_back(*p);
                }
                p++;
            } else out.push_back(*p++);
        }
        if (p >= e) return false;
        p++;
        return true;
    }
    bool val(JVal &v, int depth = 0) {
        if (depth > 200) { err = "JSON too deep"; return false; }
        ws();
        if (p >= e) { err = "unexpected end"; return false; }
        if (*p == '{') {
            v.t = JVal::Obj; p++; ws();
            if (p < e && *p == '}') { p++; return true; }
            for (;;) {
                ws(); std::string k; if (!str(k)) { err = "bad key"; return false; }
                ws(); if (p >= e || *p != ':') { err = "expected ':'"; return false; } p++;
                JVal c; if (!val(c, depth + 1)) return false;
                v.o.emplace_back(std::move(k), std::move(c));
                ws(); if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == '}') { p++; return true; }
                err = "expected ',' or '}'"; return false;
            }
        }
        if (*p == '[') {
            v.t = JVal::Arr; p++; ws();
            if (p < e && *p == ']') { p++; return true; }
            for (;;) {
                JVal c; if (!val(c, depth + 1)) return false;
                v.a.push_back(std::move(c));
                ws(); if (p < e && *p == ',') { p++; continue; }
                if (p < e && *p == ']') { p++; return true; }
                err = "expected ',' or ']'"; return false;
            }
        }
        if (*p == '"') { v.t = JVal::Str; if (!str(v.s)) { err = "bad string"; return false; } return true; }
        if (lit("true")) { v.t = JVal::Bool; v.b = true; return true; }
        if (lit("false")) { v.t = JVal::Bool; v.b = false; return true; }
        if (lit("null")) { v.t = JVal::Null; return true; }
        char *end = nullptr; double d = strtod(p, &end);
        if (end == p) { err = "bad token"; return false; }
        v.t = JVal::Num; v.n = d; p = end;
        return true;
    }
};

// untrusted JSON: a short or missing array leaves the default (*err names the field)
NodeTRS node_trs(const JVal &n, std::string *err) {
    NodeTRS o;
    auto vec = [&](const char *key, float *dst, size_t k) {
        const JVal *v = n.get(key); if (!v) return false;
        if (v->size() < k) { if (err) *err = std::string("node ") + key + " has fewer than " + std::to_string(k) + " numbers"; return false; }
        for (size_t i = 0; i < k; i++) dst[i] = (float)(*v)[i].n;
        return true;
    };
    float mm[16];
    if (vec("matrix", mm, 16)) { o.has_matrix = true; for (int c = 0; c < 4; c++) for (int rr = 0; rr < 4; rr++) o.matrix.m[rr][c] = mm[c * 4 + rr]; }
    vec("translation", o.t, 3); vec("rotation", o.r, 4); vec("scale", o.s, 3);
    return o;
}
} // namespace

M4 m4_identity() { M4 r; memset(&r, 0, sizeof r); for (int i = 0; i < 4; i++) r.m[i][i] = 1.0f; return r; }
M4 m4_mul(const M4 &a, const M4 &b) { M4 r; for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) { float s = 0.0f; for (int k = 0; k < 4; k++) s += a.m[i][k] * b.m[k][j]; r.m[i][j] = s; } return r; }
void m4_to_colmajor(const M4 &a, float out[16]) { for (int c = 0; c < 4; c++) for (int r = 0; r < 4; r++) out[c * 4 + r] = a.m[r][c]; }
static bool m4_inverse_d(const M4 &a, M4 &out) {   // Gauss-Jordan in double
    double w[4][8];
    for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) { w[i][j] = a.m[i][j]; w[i][4 + j] = i == j ? 1.0 : 0.0; }
    for (int c = 0; c < 4; c++) {
        int piv = c; for (int r = c + 1; r < 4; r++) if (fabs(w[r][c]) > fabs(w[piv][c])) piv = r;
        if (fabs(w[piv][c]) < 1e-300) return false;
        if (piv != c) for (int j = 0; j < 8; j++) std::swap(w[c][j], w[piv][j]);
        double d = w[c][c]; for (int j = 0; j < 8; j++) w[c][j] /= d;
        for (int r = 0; r < 4; r++) if (r != c) { double f = w[r][c]; if (f != 0.0) for (int j = 0; j < 8; j++) w[r][j] -= f * w[c][j]; }
    }
    for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) out.m[i][j] = (float)w[i][4 + j];
    return true;
}
// a rotation (0, 0, 0, 1) yields the identity bit for bit, so T * R * S equals the product without the rotation factor
M4 node_local(const NodeTRS &n) {
    if (n.has_matrix) return n.matrix;
    M4 t = m4_identity(), r = m4_identity(), s = m4_identity();
    for (int i = 0; i < 3; i++) t.m[i][3] = n.t[i];
    const float x = n.r[0], y = n.r[1], z = n.r[2], w = n.r[3];
    r.m[0][0] = 1 - 2 * (y * y + z * z); r.m[0][1] = 2 * (x * y - z * w); r.m[0][2] = 2 * (x * z + y * w);
    r.m[1][0] = 2 * (x * y + z * w); r.m[1][1] = 1 - 2 * (x * x + z * z); r.m[1][2] = 2 * (y * z - x * w);
    r.m[2][0] = 2 * (x * z - y * w); r.m[2][1] = 2 * (y * z + x * w); r.m[2][2] = 1 - 2 * (x * x + y * y);
    for (int i = 0; i < 3; i++) s.m[i][i] = n.s[i];
    return m4_mul(m4_mul(t, r), s);
}

static bool read_all(const std::string &path, std::vector<uint8_t> &out) {
    FILE *f = fopen(path.c_str(), "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
    out.resize(n > 0 ? (size_t)n : 0);
    size_t got = n > 0 ? fread(out.data(), 1, (size_t)n, f) : 0;
    fclose(f);
    return got == out.size();
}

// ---- texture table in PathTracer::SetScene order (PathTracer.cpp:228-408): per material base, normal, roughness, metallic, emissive; a path is
// loaded once, missing slots share the 1x1 defaults white / (128,128,255) (PathTracer.cpp:1557-1621); roughness / metallic keep the R channel (Q8)
struct TexPaths { std::string base, normal, rough, metal, emissive; };
static bool build_texture_table(HostScene &sc, const std::vector<TexPaths> &tps, std::string &err) {
    std::map<std::string, uint32_t> index_of;
    auto get_tex = [&](const std::string &p, const char *def_key, std::vector<uint8_t> def_px, bool single, uint32_t &out_idx) -> bool {
        const std::string key = p.empty() ? def_key : p;
        auto it = index_of.find(key);
        if (it != index_of.end()) { out_idx = it->second; return true; }
        HostTexture t;
        if (!p.empty()) {
            std::vector<uint8_t> rgba; uint32_t w, h;
            if (!decode_image_rgba8(p, w, h, rgba, err)) return false;
            t.width = w; t.height = h;
            if (single) { t.channels = 1; t.data.resize((size_t)w * h); for (size_t i = 0; i < (size_t)w * h; i++) t.data[i] = rgba[i * 4]; }   // R channel (Q8)
            else { t.channels = 4; t.data = std::move(rgba); }
        } else { t.width = t.height = 1; t.channels = (uint32_t)def_px.size(); t.data = def_px; }
        out_idx = (uint32_t)sc.textures.size(); index_of[key] = out_idx; sc.textures.push_back(std::move(t));
        return true;
    };
    for (size_t i = 0; i < sc.materials.size(); i++) {
        b200pt_material &m = sc.materials[i];
        if (!get_tex(tps[i].base, "EMPTY_BASECOLOR_TEXTURE", { 255, 255, 255, 255 }, false, m.BaseColorTextureIndex)) return false;
        if (!get_tex(tps[i].normal, "EMPTY_NORMAL_TEXTURE", { 128, 128, 255, 255 }, false, m.NormalTextureIndex)) return false;
        if (!get_tex(tps[i].rough, "EMPTY_ROUGHNESS_TEXTURE", { 255 }, true, m.RoughnessTextureIndex)) return false;
        if (!get_tex(tps[i].metal, "EMPTY_METALLIC_TEXTURE", { 255 }, true, m.MetallicTextureIndex)) return false;
        if (!get_tex(tps[i].emissive, "EMPTY_EMISSIVE_TEXTURE", { 255, 255, 255, 255 }, false, m.EmissiveTextureIndex)) return false;
    }
    return true;
}

// base64 payload of a "data:<mime>;base64,<payload>" URI (glTF 2.0 spec 3.6.1.1); assimp's glTF2 importer decodes these transparently
static bool decode_data_uri(const std::string &uri, std::vector<uint8_t> &out) {
    const size_t k = uri.find(";base64,");
    if (k == std::string::npos) return false;
    out.clear();
    uint32_t acc = 0; int bits = 0;
    for (size_t i = k + 8; i < uri.size(); i++) {
        const char c = uri[i];
        int v;
        if (c >= 'A' && c <= 'Z') v = c - 'A'; else if (c >= 'a' && c <= 'z') v = c - 'a' + 26; else if (c >= '0' && c <= '9') v = c - '0' + 52;
        else if (c == '+' || c == '-') v = 62; else if (c == '/' || c == '_') v = 63; else if (c == '=') break; else continue;
        acc = (acc << 6) | (uint32_t)v; bits += 6;
        if (bits >= 8) { bits -= 8; out.push_back((uint8_t)((acc >> bits) & 0xFFu)); }
    }
    return true;
}

bool load_gltf_scene(const std::string &path, HostScene &sc, std::string &err) {
    std::vector<uint8_t> text;
    if (!read_all(path, text)) { err = "cannot read " + path; return false; }
    // binary glTF (.glb, spec chapter 4): 12-byte header "glTF" | version | length, then a JSON chunk and an optional BIN chunk (= buffer 0)
    std::vector<uint8_t> glb_bin; bool is_glb = false;
    if (text.size() >= 20 && memcmp(text.data(), "glTF", 4) == 0) {
        is_glb = true;
        auto u32 = [&](size_t o) { uint32_t v; memcpy(&v, text.data() + o, 4); return v; };
        if (u32(4) != 2u) { err = "unsupported .glb container version"; return false; }
        const size_t total = std::min<size_t>(u32(8), text.size());
        size_t o = 12; std::vector<uint8_t> json;
        while (o + 8 <= total) {
            const size_t len = u32(o); const uint32_t type = u32(o + 4); o += 8;
            if (o + len > total) { err = "truncated .glb chunk"; return false; }
            if (type == 0x4E4F534Au && json.empty()) json.assign(text.begin() + (long)o, text.begin() + (long)(o + len));
            else if (type == 0x004E4942u && glb_bin.empty()) glb_bin.assign(text.begin() + (long)o, text.begin() + (long)(o + len));
            o += (len + 3u) & ~(size_t)3u;
        }
        if (json.empty()) { err = ".glb without a JSON chunk"; return false; }
        text.swap(json);
    }
    JVal g; JParser jp{ (const char *)text.data(), (const char *)text.data() + text.size(), "" };
    if (!jp.val(g) || g.t != JVal::Obj) { err = "glTF JSON parse error: " + jp.err; return false; }
    std::string base = path; { size_t k = base.find_last_of("/\\"); base = (k == std::string::npos) ? "." : base.substr(0, k); }   // AssetImporterImpl.cpp:283-284

    std::vector<std::vector<uint8_t>> buffers;
    if (const JVal *bs = g.get("buffers")) for (size_t i = 0; i < bs->size(); i++) {
        const JVal *uri = (*bs)[i].get("uri");
        buffers.emplace_back();
        if (!uri || uri->t != JVal::Str) {                                 // the BIN chunk of a .glb
            if (!is_glb || i != 0 || glb_bin.empty()) { err = "buffer without uri outside a .glb BIN chunk"; return false; }
            buffers.back() = glb_bin;
        } else if (uri->s.rfind("data:", 0) == 0) {
            if (!decode_data_uri(uri->s, buffers.back())) { err = "unsupported data: URI encoding (base64 expected)"; return false; }
        } else if (!read_all(base + "/" + uri->s, buffers.back())) { err = "cannot read buffer " + uri->s; return false; }
    }
    const JVal *accs = g.get("accessors"), *views = g.get("bufferViews");
    auto accessor = [&](int idx, int want_comps, std::vector<float> *fout, std::vector<uint32_t> *uout, size_t &count) -> bool {
        if (!accs || !views || idx < 0 || (size_t)idx >= accs->size()) { err = "bad accessor index"; return false; }
        const JVal &a = (*accs)[idx];
        auto to_sz = [](double v) { return (v >= 0.0 && v < 4294967296.0) ? (size_t)v : (size_t)-1; };   // untrusted JSON numbers: no UB casts, no 64-bit wrap
        int ct = (int)a.num("componentType", 0); count = to_sz(a.num("count", 0));
        if (count == (size_t)-1) { err = "bad accessor count"; return false; }
        const JVal *ty = a.get("type"); if (!ty) { err = "accessor without type"; return false; }
        int nc = ty->s == "SCALAR" ? 1 : ty->s == "VEC2" ? 2 : ty->s == "VEC3" ? 3 : ty->s == "VEC4" ? 4 : 0;
        if (nc != want_comps) { err = "unexpected accessor type " + ty->s; return false; }
        int bvi = (int)a.num("bufferView", -1); if (bvi < 0 || (size_t)bvi >= views->size()) { err = "sparse/empty accessors not supported"; return false; }
        const JVal &bv = (*views)[bvi];
        const size_t off_v = to_sz(bv.num("byteOffset", 0)), off_a = to_sz(a.num("byteOffset", 0));
        if (off_v == (size_t)-1 || off_a == (size_t)-1) { err = "bad byteOffset"; return false; }
        size_t off = off_v + off_a;
        int csz = (ct == 5120 || ct == 5121) ? 1 : (ct == 5122 || ct == 5123) ? 2 : (ct == 5125 || ct == 5126) ? 4 : 0;
        if (!csz) { err = "bad componentType"; return false; }
        size_t stride = to_sz(bv.num("byteStride", 0)); if (!stride) stride = (size_t)csz * nc;
        int bi = (int)bv.num("buffer", 0); if ((size_t)bi >= buffers.size()) { err = "bad buffer index"; return false; }
        const std::vector<uint8_t> &buf = buffers[bi];
        {   // all in division form: count / offsets come from untrusted JSON doubles and the products can wrap in 64 bits
            const size_t elem = (size_t)csz * nc;
            if (stride < elem || stride > 4096) { err = "bad byteStride"; return false; }
            if (count && (off > buf.size() || elem > buf.size() - off || count - 1 > (buf.size() - off - elem) / stride)) { err = "accessor out of range"; return false; }
        }
        const bool norm = a.get("normalized") && a.get("normalized")->b;
        if (fout) fout->resize(count * nc);
        if (uout) uout->resize(count * nc);
        for (size_t i = 0; i < count; i++) for (int c = 0; c < nc; c++) {
            const uint8_t *p = &buf[off + i * stride + (size_t)c * csz];
            double v = 0; uint32_t u = 0;
            switch (ct) {
            case 5120: { int8_t x; memcpy(&x, p, 1); v = x; u = (uint32_t)x; if (norm) v = std::max(x / 127.0, -1.0); } break;
            case 5121: { uint8_t x = *p; v = x; u = x; if (norm) v = x / 255.0; } break;
            case 5122: { int16_t x; memcpy(&x, p, 2); v = x; u = (uint32_t)x; if (norm) v = std::max(x / 32767.0, -1.0); } break;
            case 5123: { uint16_t x; memcpy(&x, p, 2); v = x; u = x; if (norm) v = x / 65535.0; } break;
            case 5125: { uint32_t x; memcpy(&x, p, 4); v = x; u = x; } break;
            case 5126: { float x; memcpy(&x, p, 4); v = x; u = (uint32_t)x; } break;
            }
            if (fout) (*fout)[i * nc + c] = (float)v;
            if (uout) (*uout)[i * nc + c] = u;
        }
        return true;
    };

    // Accessors of the animation data (skins, JOINTS_n / WEIGHTS_n, morph targets, animations).  Unlike the geometry's accessor above, these
    // may be sparse or have no bufferView (zeros), and a failure only sets aerr: animation data never fails a load.  Values are decoded as the
    // accessor says (float, or normalized integers); expect != SIZE_MAX: the element count the caller needs.
    auto elems = [&](double bvd, double offd, int ct, int nc, size_t count, bool norm, double *out, std::string &aerr) -> bool {
        auto to_sz = [](double v) { return (v >= 0.0 && v < 4294967296.0) ? (size_t)v : (size_t)-1; };
        if (!views || !(bvd >= 0.0 && bvd < (double)views->size())) { aerr = "bad bufferView index"; return false; }
        const JVal &bv = (*views)[(size_t)bvd];
        const size_t off_v = to_sz(bv.num("byteOffset", 0)), off_a = to_sz(offd);
        if (off_v == (size_t)-1 || off_a == (size_t)-1) { aerr = "bad byteOffset"; return false; }
        const size_t off = off_v + off_a;
        const int csz = (ct == 5120 || ct == 5121) ? 1 : (ct == 5122 || ct == 5123) ? 2 : (ct == 5125 || ct == 5126) ? 4 : 0;
        if (!csz) { aerr = "bad componentType"; return false; }
        const size_t elem = (size_t)csz * nc;
        size_t stride = to_sz(bv.num("byteStride", 0)); if (!stride) stride = elem;
        if (stride < elem || stride > 4096) { aerr = "bad byteStride"; return false; }
        const double bid = bv.num("buffer", 0);
        if (!(bid >= 0.0 && bid < (double)buffers.size())) { aerr = "bad buffer index"; return false; }
        const std::vector<uint8_t> &buf = buffers[(size_t)bid];
        if (count && (off > buf.size() || elem > buf.size() - off || count - 1 > (buf.size() - off - elem) / stride)) { aerr = "accessor out of range"; return false; }
        for (size_t i = 0; i < count; i++) for (int c = 0; c < nc; c++) {
            const uint8_t *p = &buf[off + i * stride + (size_t)c * csz];
            double v = 0;
            switch (ct) {
            case 5120: { int8_t x; memcpy(&x, p, 1); v = norm ? std::max(x / 127.0, -1.0) : x; } break;
            case 5121: { uint8_t x = *p; v = norm ? x / 255.0 : x; } break;
            case 5122: { int16_t x; memcpy(&x, p, 2); v = norm ? std::max(x / 32767.0, -1.0) : x; } break;
            case 5123: { uint16_t x; memcpy(&x, p, 2); v = norm ? x / 65535.0 : x; } break;
            case 5125: { uint32_t x; memcpy(&x, p, 4); v = x; } break;
            case 5126: { float x; memcpy(&x, p, 4); v = x; } break;
            }
            out[i * nc + c] = v;
        }
        return true;
    };
    auto anim_accessor = [&](const JVal *idxv, int want_comps, size_t expect, std::vector<double> &out, size_t &count, std::string &aerr,
                             int *ct_out = nullptr, bool *norm_out = nullptr) -> bool {
        if (!idxv || idxv->t != JVal::Num || !accs || !(idxv->n >= 0.0 && idxv->n < (double)accs->size())) { aerr = "bad accessor index"; return false; }
        const JVal &a = (*accs)[(size_t)idxv->n];
        const double cd = a.num("count", -1.0);
        if (!(cd >= 1.0 && cd <= (double)(1u << 26)) || cd != std::floor(cd)) { aerr = "bad accessor count"; return false; }
        count = (size_t)cd;
        if (expect != (size_t)-1 && count != expect) { aerr = "accessor count mismatch"; return false; }
        const JVal *ty = a.get("type"); const std::string ts = ty && ty->t == JVal::Str ? ty->s : "";
        const int nc = ts == "SCALAR" ? 1 : ts == "VEC2" ? 2 : ts == "VEC3" ? 3 : ts == "VEC4" ? 4 : ts == "MAT4" ? 16 : 0;
        if (!nc || nc != want_comps) { aerr = "unexpected accessor type " + ts; return false; }
        const int ct = (int)a.num("componentType", 0);
        const bool norm = a.get("normalized") && a.get("normalized")->b;
        if (ct_out) *ct_out = ct;
        if (norm_out) *norm_out = norm;
        const JVal *bvv = a.get("bufferView"), *sp = a.get("sparse");
        if (!bvv && !sp) { aerr = "accessor without bufferView or sparse"; return false; }
        out.assign(count * nc, 0.0);
        if (bvv && !elems(bvv->n, a.num("byteOffset", 0), ct, nc, count, norm, out.data(), aerr)) return false;
        if (sp) {                                                          // glTF 2.0 3.6.2.3: values replace the elements at the given indices
            const double sc = sp->num("count", -1.0);
            const JVal *si = sp->get("indices"), *sv = sp->get("values");
            if (!(sc >= 1.0 && sc <= (double)count) || sc != std::floor(sc) || !si || !sv) { aerr = "bad sparse accessor"; return false; }
            const size_t m = (size_t)sc;
            const int ict = (int)si->num("componentType", 0);
            if (ict != 5121 && ict != 5123 && ict != 5125) { aerr = "bad sparse index componentType"; return false; }
            std::vector<double> ix(m), vals(m * nc);
            if (!elems(si->num("bufferView", -1), si->num("byteOffset", 0), ict, 1, m, false, ix.data(), aerr)) return false;
            if (!elems(sv->num("bufferView", -1), sv->num("byteOffset", 0), ct, nc, m, norm, vals.data(), aerr)) return false;
            for (size_t k = 0; k < m; k++) {
                if (!(ix[k] < (double)count)) { aerr = "sparse index out of range"; return false; }
                for (int c = 0; c < nc; c++) out[(size_t)ix[k] * nc + c] = vals[k * nc + c];
            }
        }
        for (double v : out) if (!std::isfinite(v) || std::fabs(v) > 3.4e38) { aerr = "non-finite value"; return false; }
        return true;
    };
    auto anim = std::make_shared<HostAnimation>();

    // ---- meshes: one per primitive (AssetImporterImpl.cpp:121-218)
    std::vector<std::vector<uint32_t>> prims_of_mesh; std::vector<int> mesh_material;
    if (const JVal *ms = g.get("meshes")) for (size_t mi = 0; mi < ms->size(); mi++) {
        prims_of_mesh.emplace_back();
        const JVal *prs = (*ms)[mi].get("primitives"); if (!prs) continue;
        for (size_t pi = 0; pi < prs->size(); pi++) {
            const JVal &p = (*prs)[pi];
            const int mode = (int)p.num("mode", 4);
            if (mode < 4 || mode > 6) { err = "only TRIANGLES / TRIANGLE_STRIP / TRIANGLE_FAN primitives are supported"; return false; }
            const JVal *at = p.get("attributes"); if (!at || !at->has("POSITION")) { err = "primitive without POSITION"; return false; }
            std::vector<float> pos, nrm, uv; size_t n = 0, nn = 0, nu = 0;
            if (!accessor((int)at->num("POSITION", -1), 3, &pos, nullptr, n)) return false;
            const bool has_nrm = at->has("NORMAL");
            if (has_nrm && (!accessor((int)at->num("NORMAL", -1), 3, &nrm, nullptr, nn) || nn != n)) { if (err.empty()) err = "NORMAL count mismatch"; return false; }
            const bool has_uv = at->has("TEXCOORD_0");
            if (has_uv && (!accessor((int)at->num("TEXCOORD_0", -1), 2, &uv, nullptr, nu) || nu != n)) { if (err.empty()) err = "TEXCOORD_0 count mismatch"; return false; }
            HostMesh hm; hm.vertices.resize(n);
            if (const JVal *nm = (*ms)[mi].get("name")) hm.name = nm->s;
            if (p.has("indices")) { size_t ni = 0; if (!accessor((int)p.num("indices", -1), 1, nullptr, &hm.indices, ni)) return false; }
            else { hm.indices.resize(n); for (size_t i = 0; i < n; i++) hm.indices[i] = (uint32_t)i; }
            if (mode != 4) {                                              // assimp's glTF2 importer expands strips and fans into triangle faces
                std::vector<uint32_t> src; src.swap(hm.indices);
                const size_t nf = src.size() >= 3 ? src.size() - 2 : 0;
                for (size_t f = 0; f < nf; f++) {
                    if (mode == 5) { if ((f + 1) % 2 == 0) { hm.indices.push_back(src[f + 1]); hm.indices.push_back(src[f]); } else { hm.indices.push_back(src[f]); hm.indices.push_back(src[f + 1]); } hm.indices.push_back(src[f + 2]); }   // same orientation for every triangle
                    else { hm.indices.push_back(src[0]); hm.indices.push_back(src[f + 1]); hm.indices.push_back(src[f + 2]); }
                }
            }
            hm.indices.resize(hm.indices.size() / 3 * 3);
            for (uint32_t ix : hm.indices) if (ix >= n) { err = "index out of range"; return false; }
            if (hm.indices.empty() || n == 0) { err = "primitive without triangles"; return false; }
            if (!has_nrm) {
                // aiProcess_GenNormals (AssetImporterImpl.cpp:82-97) = assimp 6.0.2 GenFaceNormalsProcess (from upstream knowledge, SURVEY 8c):
                // every face writes NormalizeSafe(cross(v1 - v0, v2 - v0)) to its three vertices, so a shared vertex keeps the normal of the
                // LAST face that uses it (assimp does not split vertices here); a vertex no face references stays (0, 0, 0).
                nrm.assign(n * 3, 0.0f);
                for (size_t f = 0; f + 2 < hm.indices.size(); f += 3) {
                    const float *a = &pos[hm.indices[f] * 3], *b = &pos[hm.indices[f + 1] * 3], *c = &pos[hm.indices[f + 2] * 3];
                    const float e1[3] = { b[0] - a[0], b[1] - a[1], b[2] - a[2] }, e2[3] = { c[0] - a[0], c[1] - a[1], c[2] - a[2] };
                    float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
                    const float len = sqrtf(nx * nx + ny * ny + nz * nz);
                    if (len > 0.0f) { nx /= len; ny /= len; nz /= len; }
                    for (int k = 0; k < 3; k++) { float *o = &nrm[hm.indices[f + k] * 3]; o[0] = nx; o[1] = ny; o[2] = nz; }
                }
            }
            for (size_t i = 0; i < n; i++) {
                b200pt_vertex &v = hm.vertices[i];
                v.Position[0] = pos[i * 3]; v.Position[1] = pos[i * 3 + 1]; v.Position[2] = pos[i * 3 + 2];
                const float nx = nrm[i * 3], ny = nrm[i * 3 + 1], nz = nrm[i * 3 + 2];
                const float inv = 1.0f / sqrtf(nx * nx + ny * ny + nz * nz);              // glm::normalize (:165)
                v.Normal[0] = nx * inv; v.Normal[1] = ny * inv; v.Normal[2] = nz * inv;
                v.TexCoord[0] = has_uv ? uv[i * 2] : 0.0f; v.TexCoord[1] = has_uv ? uv[i * 2 + 1] : 0.0f;   // importer flip + FlipUVs = identity
            }
            {   // what a pose of this primitive needs (skins, morph targets); problems go to ap.err
                AnimPrim ap; try { ap.gltf_mesh = (int)mi; ap.count = (uint32_t)n; ap.gen_normals = !has_nrm;
                std::vector<std::vector<double>> js, ws;
                for (uint32_t s = 0; s < 16 && ap.err.empty(); s++) {
                    const std::string jn = "JOINTS_" + std::to_string(s), wn = "WEIGHTS_" + std::to_string(s);
                    const JVal *ja = at->get(jn.c_str()), *wa = at->get(wn.c_str());
                    if (!ja && !wa) break;
                    std::vector<double> j, w; size_t c = 0; int ct = 0; bool nm = false;
                    if (!ja || !wa) { ap.err = jn + " / " + wn + " not paired"; break; }
                    if (!anim_accessor(ja, 4, n, j, c, ap.err, &ct)) { ap.err = jn + ": " + ap.err; break; }
                    if (ct != 5121 && ct != 5123) { ap.err = jn + ": joints must be unsigned byte or unsigned short"; break; }
                    if (!anim_accessor(wa, 4, n, w, c, ap.err, &ct, &nm)) { ap.err = wn + ": " + ap.err; break; }
                    if (!(ct == 5126 || ((ct == 5121 || ct == 5123) && nm))) { ap.err = wn + ": weights must be float or normalized unsigned byte / short"; break; }
                    js.push_back(std::move(j)); ws.push_back(std::move(w));
                }
                // a set the loop did not read (a 17th, or one after a gap in the numbering) would silently lose its influences
                for (size_t k = 0; k < at->o.size() && ap.err.empty(); k++)
                    for (const char *pre : { "JOINTS_", "WEIGHTS_" }) {
                        const std::string &name = at->o[k].first;
                        if (ap.err.empty() && !name.compare(0, strlen(pre), pre) && strtoul(name.c_str() + strlen(pre), nullptr, 10) >= js.size())
                            ap.err = name + ": more than 16 JOINTS_n / WEIGHTS_n sets, or a gap in their numbering";
                    }
                if (ap.err.empty() && !js.empty()) {
                    ap.sets = (uint32_t)js.size();
                    ap.joints.resize(n * 4 * ap.sets); ap.weights.resize(n * 4 * ap.sets);
                    for (size_t i = 0; i < n; i++) for (uint32_t s = 0; s < ap.sets; s++) for (int k = 0; k < 4; k++) {
                        ap.joints[(i * ap.sets + s) * 4 + k] = (uint32_t)js[s][i * 4 + k];
                        ap.weights[(i * ap.sets + s) * 4 + k] = (float)ws[s][i * 4 + k];
                    }
                }
                const JVal *tg = p.get("targets");
                if (tg && tg->t == JVal::Arr && tg->size()) {
                    ap.targets = (uint32_t)std::min<size_t>(tg->size(), 256);
                    if (tg->size() > 256) ap.err = "more than 256 morph targets";
                    struct { const char *key; int nc; std::vector<float> *dst; } attrs[3] = { { "POSITION", 3, &ap.dpos }, { "NORMAL", 3, &ap.dnrm }, { "TEXCOORD_0", 2, &ap.duv } };
                    for (uint32_t t = 0; t < ap.targets && ap.err.empty(); t++) {
                        const JVal &tj = (*tg)[t];
                        for (auto &A : attrs) {
                            const JVal *ix = tj.get(A.key); if (!ix) continue;         // TANGENT / COLOR_n: no field in b200pt_vertex
                            std::vector<double> d; size_t c = 0;
                            if (!anim_accessor(ix, A.nc, n, d, c, ap.err)) { ap.err = std::string("morph target ") + A.key + ": " + ap.err; break; }
                            if (A.dst->empty()) A.dst->assign((size_t)ap.targets * n * A.nc, 0.0f);
                            for (size_t k = 0; k < n * A.nc; k++) (*A.dst)[(size_t)t * n * A.nc + k] = (float)d[k];
                        }
                    }
                }
                if (ap.sets || ap.targets) {
                    ap.rest.resize(n * 8);
                    for (size_t i = 0; i < n; i++) {
                        for (int k = 0; k < 3; k++) { ap.rest[i * 8 + k] = pos[i * 3 + k]; ap.rest[i * 8 + 3 + k] = has_nrm ? nrm[i * 3 + k] : 0.0f; }
                        ap.rest[i * 8 + 6] = hm.vertices[i].TexCoord[0]; ap.rest[i * 8 + 7] = hm.vertices[i].TexCoord[1];
                    }
                    if (!has_nrm) {
                        ap.last_face.assign(n, UINT32_MAX);
                        for (size_t f = 0; f + 2 < hm.indices.size(); f += 3) for (int k = 0; k < 3; k++) ap.last_face[hm.indices[f + k]] = (uint32_t)(f / 3);
                    }
                }
                } catch (const std::bad_alloc &) { ap = AnimPrim(); ap.gltf_mesh = (int)mi; ap.count = (uint32_t)n; ap.err = "out of memory reading the skin / morph data"; }
                anim->prims.push_back(std::move(ap));
            }
            prims_of_mesh.back().push_back((uint32_t)sc.meshes.size());
            mesh_material.push_back(p.has("material") ? (int)p.num("material", 0) : -1);
            sc.meshes.push_back(std::move(hm));
        }
    }
    if (sc.meshes.empty()) { err = "No meshes found in scene"; return false; }                // PathTracer.cpp:180

    // ---- materials (:353-455)
    const JVal *mats = g.get("materials"), *texs = g.get("textures"), *imgs = g.get("images");
    size_t nmat = mats ? mats->size() : 0;
    bool need_default = false; for (int m : mesh_material) if (m < 0) need_default = true;
    std::vector<TexPaths> tps;
    bool embedded_image = false;
    auto tex_path = [&](const JVal *ti) -> std::string {
        if (!ti || !texs) return "";
        int idx = (int)ti->num("index", -1); if (idx < 0 || (size_t)idx >= texs->size()) return "";
        int src = (int)(*texs)[idx].num("source", -1); if (src < 0 || !imgs || (size_t)src >= imgs->size()) return "";
        const JVal *uri = (*imgs)[src].get("uri");
        if (!uri || uri->s.rfind("data:", 0) == 0) { embedded_image = true; return ""; }         // bufferView / data: images: the reference only loads texture FILES (:287-328)
        return base + "/" + uri->s;                                                            // :287-328
    };
    for (size_t i = 0; i < nmat + (need_default ? 1 : 0); i++) {
        static const JVal empty_obj = [] { JVal v; v.t = JVal::Obj; return v; }();
        const JVal &m = i < nmat ? (*mats)[i] : empty_obj;
        const JVal *pbr = m.get("pbrMetallicRoughness"); if (!pbr) pbr = &empty_obj;
        const JVal *ext = m.get("extensions"); if (!ext) ext = &empty_obj;
        b200pt_material o; memset(&o, 0, sizeof o);
        for (int k = 0; k < 3; k++) { o.BaseColor[k] = 1.0f; o.SpecularColor[k] = 1.0f; o.MediumColor[k] = 1.0f; }
        if (const JVal *bc = pbr->get("baseColorFactor")) for (int k = 0; k < 3; k++) o.BaseColor[k] = (float)(*bc)[k].n;
        float strength = 1.0f; if (const JVal *es = ext->get("KHR_materials_emissive_strength")) strength = (float)es->num("emissiveStrength", 1.0);
        if (const JVal *ef = m.get("emissiveFactor")) for (int k = 0; k < 3; k++) o.EmissiveColor[k] = (float)(*ef)[k].n * strength;
        if (const JVal *sp = ext->get("KHR_materials_specular")) if (const JVal *c = sp->get("specularColorFactor")) for (int k = 0; k < 3; k++) o.SpecularColor[k] = (float)(*c)[k].n;
        o.Metallic = (float)pbr->num("metallicFactor", 1.0);        // glTF default 1.0: assimp always sets AI_MATKEY_METALLIC_FACTOR
        o.Roughness = (float)pbr->num("roughnessFactor", 1.0);
        o.IOR = 1.5f; if (const JVal *e = ext->get("KHR_materials_ior")) o.IOR = (float)e->num("ior", 1.5);
        if (const JVal *e = ext->get("KHR_materials_transmission")) o.Transmission = (float)e->num("transmissionFactor", 0.0);
        if (const JVal *e = ext->get("KHR_materials_anisotropy")) { o.Anisotropy = (float)e->num("anisotropyStrength", 0.0); o.AnisotropyRotation = (float)e->num("anisotropyRotation", 0.0) * (180.0f / 3.14159265358979323846f); }
        sc.materials.push_back(o);
        const JVal *nm = m.get("name"); sc.material_names.push_back(nm ? nm->s : (i < nmat ? "" : "DefaultMaterial"));
        TexPaths tp; tp.base = tex_path(pbr->get("baseColorTexture")); tp.normal = tex_path(m.get("normalTexture"));
        tp.rough = tp.metal = tex_path(pbr->get("metallicRoughnessTexture")); tp.emissive = tex_path(m.get("emissiveTexture"));
        tps.push_back(tp);
    }
    if (embedded_image) { err = "embedded (bufferView / data: URI) textures are not supported: the reference loads textures from files next to the model only"; return false; }
    if (!build_texture_table(sc, tps, err)) return false;

    // ---- nodes -> instances + first camera (:220-262, :547-642)
    const JVal *nodes = g.get("nodes"), *scenes = g.get("scenes"), *cams = g.get("cameras");
    M4 flip = m4_identity(); flip.m[1][1] = -1.0f;
    bool have_cam = false;
    struct Item { int node; M4 parent; };
    std::vector<Item> order;
    std::vector<int> roots;
    if (scenes && scenes->size()) { const JVal &s = (*scenes)[(size_t)g.num("scene", 0) < scenes->size() ? (size_t)g.num("scene", 0) : 0]; if (const JVal *ns = s.get("nodes")) for (size_t i = 0; i < ns->size(); i++) roots.push_back((int)(*ns)[i].n); }
    std::vector<std::pair<int, M4>> stack;   // explicit DFS preserving child order
    for (size_t ri = roots.size(); ri-- > 0;) stack.push_back({ roots[ri], m4_identity() });
    const uint32_t default_mat = (uint32_t)sc.materials.size() - 1;
    size_t guard = 0;
    while (!stack.empty()) {
        auto [ni, parent] = stack.back(); stack.pop_back();
        if (!nodes || ni < 0 || (size_t)ni >= nodes->size() || ++guard > 10000000) { err = "bad node graph"; return false; }
        const JVal &n = (*nodes)[ni];
        const M4 world = m4_mul(parent, node_local(node_trs(n, nullptr)));
        if (n.has("mesh")) {
            size_t mi = (size_t)n.num("mesh", 0);
            if (mi < prims_of_mesh.size()) for (uint32_t pm : prims_of_mesh[mi]) {
                b200pt_instance in; m4_to_colmajor(m4_mul(flip, world), in.Transform);
                in.MeshIndex = pm; in.MaterialIndex = mesh_material[pm] < 0 ? default_mat : (uint32_t)mesh_material[pm];
                if (in.MaterialIndex >= sc.materials.size()) { err = "Mesh instance has invalid material index"; return false; }
                sc.instances.push_back(in);
                anim->instance_node.push_back(ni);
            }
        }
        if (n.has("camera") && !have_cam && (int)n.num("camera", -1) == 0 && cams && cams->size()) {
            M4 local = m4_identity(); local.m[1][1] = -1.0f;      // columns right(1,0,0), up(0,-1,0), -lookAt(0,0,1)
            M4 fin = m4_mul(m4_mul(flip, world), local), view;
            if (!m4_inverse_d(fin, view)) { err = "singular camera transform"; return false; }
            m4_to_colmajor(view, sc.camera_view);
            double asp = 0.0; if (const JVal *pp = (*cams)[0].get("perspective")) asp = pp->num("aspectRatio", 0.0);
            sc.camera_aspect = asp > 0.0 ? (float)asp : 1.0f;
            have_cam = true;
        }
        if (const JVal *ch = n.get("children")) for (size_t ci = ch->size(); ci-- > 0;) stack.push_back({ (int)(*ch)[ci].n, world });
    }
    if (!have_cam) {   // PathTracer.cpp:171-178: lookAt((0,0,5),(0,0,0),(0,1,0)), aspect 16/9
        M4 v = m4_identity(); v.m[2][3] = -5.0f; m4_to_colmajor(v, sc.camera_view); sc.camera_aspect = 16.0f / 9.0f;
    }
    if (sc.instances.empty()) { err = "scene has no mesh instances"; return false; }

    // ---- animation data: node graph, skins, morph weights, animations.  Nothing below fails the load.
    HostAnimation &A = *anim;
    try {
        auto index = [](const JVal *v, size_t n) { return (v && v->t == JVal::Num && v->n >= 0.0 && v->n < (double)n && v->n == std::floor(v->n)) ? (int)v->n : -1; };
        const size_t nn = nodes ? nodes->size() : 0, nskin = g.get("skins") ? g.get("skins")->size() : 0;
        A.roots = roots;
        A.nodes.resize(nn);
        const JVal *ms = g.get("meshes");
        A.mesh_weights.resize(prims_of_mesh.size()); A.mesh_targets.assign(prims_of_mesh.size(), 0);
        for (size_t mi = 0; mi < prims_of_mesh.size(); mi++) {
            for (size_t k = 0; k < prims_of_mesh[mi].size(); k++) {
                const AnimPrim &ap = A.prims[prims_of_mesh[mi][k]];
                if (k == 0) A.mesh_targets[mi] = ap.targets;
                else if (ap.targets != A.mesh_targets[mi] && A.err.empty()) A.err = "mesh " + std::to_string(mi) + ": primitives with different morph target counts";
            }
            if (const JVal *w = (*ms)[mi].get("weights")) for (size_t k = 0; k < w->size(); k++) A.mesh_weights[mi].push_back((float)(*w)[k].n);
            if (!A.mesh_weights[mi].empty() && A.mesh_weights[mi].size() != A.mesh_targets[mi] && A.err.empty()) A.err = "mesh " + std::to_string(mi) + ": weights count differs from its morph targets";
        }
        for (size_t i = 0; i < nn; i++) {
            const JVal &n = (*nodes)[i]; AnimNode &an = A.nodes[i];
            std::string e; an.trs = node_trs(n, &e);
            if (!e.empty() && A.err.empty()) A.err = "node " + std::to_string(i) + ": " + e;
            if (const JVal *ch = n.get("children")) for (size_t c = 0; c < ch->size(); c++) {
                const int ci = index(&(*ch)[c], nn);
                if (ci < 0 && A.err.empty()) A.err = "node " + std::to_string(i) + ": child index out of range";
                if (ci >= 0) an.children.push_back(ci);
            }
            if (n.has("mesh")) an.mesh = index(n.get("mesh"), prims_of_mesh.size());
            if (n.has("skin")) { an.skin = index(n.get("skin"), nskin); if (an.skin < 0 && A.err.empty()) A.err = "node " + std::to_string(i) + ": skin index out of range"; }
            if (const JVal *w = n.get("weights")) {
                an.has_weights = true;
                for (size_t k = 0; k < w->size(); k++) an.weights.push_back((float)(*w)[k].n);
                if (an.mesh >= 0 && an.weights.size() != A.mesh_targets[an.mesh] && A.err.empty()) A.err = "node " + std::to_string(i) + ": weights count differs from its mesh's morph targets";
            }
        }
        if (const JVal *sk = g.get("skins")) for (size_t s = 0; s < sk->size(); s++) {
            AnimSkin S; const JVal &sj = (*sk)[s];
            if (const JVal *js = sj.get("joints")) for (size_t k = 0; k < js->size(); k++) {
                const int j = index(&(*js)[k], nn);
                if (j < 0 && S.err.empty()) S.err = "skin " + std::to_string(s) + ": joint index out of range";
                S.joints.push_back(j < 0 ? 0 : j);
            }
            if (S.joints.empty() && S.err.empty()) S.err = "skin " + std::to_string(s) + " has no joints";
            S.inverse_bind.assign(S.joints.size(), m4_identity());
            if (const JVal *ib = sj.get("inverseBindMatrices"); ib && S.err.empty()) {
                std::vector<double> d; size_t c = 0; std::string e;
                if (!anim_accessor(ib, 16, S.joints.size(), d, c, e)) S.err = "skin " + std::to_string(s) + " inverseBindMatrices: " + e;
                else for (size_t k = 0; k < S.joints.size(); k++) for (int cc = 0; cc < 4; cc++) for (int r = 0; r < 4; r++) S.inverse_bind[k].m[r][cc] = (float)d[k * 16 + cc * 4 + r];
            }
            A.skins.push_back(std::move(S));
        }
        if (const JVal *as = g.get("animations")) for (size_t ai = 0; ai < as->size(); ai++) {
            const JVal &aj = (*as)[ai]; AnimClip C;
            if (const JVal *nm = aj.get("name")) C.name = nm->s;
            const JVal *smp = aj.get("samplers"), *chs = aj.get("channels");
            const size_t nsmp = smp ? smp->size() : 0;
            for (size_t si = 0; si < nsmp; si++) {
                const JVal &s = (*smp)[si]; AnimSampler S; std::string e;
                const JVal *ip = s.get("interpolation");
                const std::string it = ip && ip->t == JVal::Str ? ip->s : "LINEAR";
                S.interp = it == "STEP" ? INTERP_STEP : it == "CUBICSPLINE" ? INTERP_CUBIC : INTERP_LINEAR;
                if (it != "STEP" && it != "LINEAR" && it != "CUBICSPLINE") e = "unknown interpolation " + it;
                std::vector<double> in, out; size_t ni = 0, no = 0;
                const JVal *oacc = (accs && s.get("output") && index(s.get("output"), accs->size()) >= 0) ? &(*accs)[(size_t)s.get("output")->n] : nullptr;
                const JVal *oty = oacc ? oacc->get("type") : nullptr;
                const std::string ots = oty && oty->t == JVal::Str ? oty->s : "";
                const int onc = ots == "SCALAR" ? 1 : ots == "VEC3" ? 3 : ots == "VEC4" ? 4 : 0;
                if (e.empty() && !anim_accessor(s.get("input"), 1, (size_t)-1, in, ni, e)) e = "input: " + e;
                if (e.empty() && !onc) e = "output: unexpected accessor type " + ots;
                if (e.empty() && !anim_accessor(s.get("output"), onc, (size_t)-1, out, no, e)) e = "output: " + e;
                if (e.empty()) for (size_t k = 1; k < ni; k++) if (!(in[k] > in[k - 1])) { e = "input times do not increase"; break; }
                if (e.empty()) {
                    S.input.assign(in.begin(), in.end()); S.output.assign(out.begin(), out.end());
                    for (size_t k = 1; k < ni && e.empty(); k++) if (!(S.input[k] > S.input[k - 1])) e = "input times do not increase in float";
                    const size_t per_key = S.interp == INTERP_CUBIC ? 3 : 1;
                    if (e.empty() && (no % (ni * per_key))) e = "output count is not a multiple of the input count";
                    S.comps = e.empty() ? (uint32_t)(no / (ni * per_key) * onc) : 0;
                }
                if (!e.empty()) S.err = "sampler " + std::to_string(si) + ": " + e;
                C.samplers.push_back(std::move(S));
            }
            if (chs) for (size_t ci = 0; ci < chs->size() && C.err.empty(); ci++) {
                const JVal &c = (*chs)[ci]; const JVal *tg = c.get("target");
                const JVal *pj = tg ? tg->get("path") : nullptr;
                const std::string path = pj && pj->t == JVal::Str ? pj->s : "";
                AnimChannel ch;
                ch.path = path == "translation" ? PATH_T : path == "rotation" ? PATH_R : path == "scale" ? PATH_S : path == "weights" ? PATH_W : -1;
                if (ch.path < 0) continue;                                 // KHR_animation_pointer and other extensions: not posed
                if (!tg->has("node")) continue;                            // glTF 2.0 5.5.2.1: a channel without a node is ignored
                ch.node = index(tg->get("node"), nn); ch.sampler = index(c.get("sampler"), nsmp);
                const std::string where = "channel " + std::to_string(ci) + ": ";
                if (ch.node < 0) { C.err = where + "target node out of range"; break; }
                if (ch.sampler < 0) { C.err = where + "sampler index out of range"; break; }
                const AnimSampler &S = C.samplers[ch.sampler];
                if (!S.err.empty()) { C.err = where + S.err; break; }
                const AnimNode &an = A.nodes[ch.node];
                if (ch.path != PATH_W && an.trs.has_matrix) { C.err = where + "animates a node that has a matrix"; break; }
                const uint32_t want = ch.path == PATH_R ? 4 : ch.path == PATH_W ? (an.mesh >= 0 ? A.mesh_targets[an.mesh] : 0) : 3;
                if (!want || S.comps != want) { C.err = where + "output size does not match the path"; break; }
                C.channels.push_back(ch);
            }
            animation_range(C, &C.t0, &C.t1);
            A.clips.push_back(std::move(C));
        }
        finalize_animation(A, sc);
    } catch (const std::bad_alloc &) {
        if (A.err.empty()) A.err = "out of memory reading the animation data";
    }
    sc.animation = anim;
    return true;
}

bool scene_from_desc(const b200pt_scene_desc *d, HostScene &sc, std::string &err) {
    if (!d || !d->meshes || !d->materials || !d->textures || !d->instances || !d->mesh_count || !d->material_count || !d->texture_count || !d->instance_count) { err = "scene description has empty arrays"; return false; }
    for (uint32_t i = 0; i < d->mesh_count; i++) {
        const b200pt_mesh &m = d->meshes[i];
        if (!m.vertices || !m.indices || !m.vertex_count || m.index_count < 3) { err = "empty mesh"; return false; }
        HostMesh hm; hm.vertices.assign(m.vertices, m.vertices + m.vertex_count); hm.indices.assign(m.indices, m.indices + m.index_count / 3 * 3);
        for (uint32_t ix : hm.indices) if (ix >= m.vertex_count) { err = "index out of range"; return false; }
        sc.meshes.push_back(std::move(hm));
    }
    sc.materials.assign(d->materials, d->materials + d->material_count);
    sc.material_names.assign(d->material_count, "");
    for (uint32_t i = 0; i < d->texture_count; i++) {
        const b200pt_texture &t = d->textures[i];
        if (!t.data || !t.width || !t.height || (t.channels != 1 && t.channels != 4)) { err = "bad texture"; return false; }
        HostTexture ht; ht.width = t.width; ht.height = t.height; ht.channels = t.channels; ht.data.assign(t.data, t.data + (size_t)t.width * t.height * t.channels);
        sc.textures.push_back(std::move(ht));
    }
    for (const b200pt_material &m : sc.materials) {
        const uint32_t ix[5] = { m.BaseColorTextureIndex, m.NormalTextureIndex, m.RoughnessTextureIndex, m.MetallicTextureIndex, m.EmissiveTextureIndex };
        for (uint32_t k : ix) if (k >= d->texture_count) { err = "material texture index out of range"; return false; }
    }
    sc.instances.assign(d->instances, d->instances + d->instance_count);
    for (const b200pt_instance &in : sc.instances) if (in.MeshIndex >= d->mesh_count || in.MaterialIndex >= d->material_count) { err = "Mesh instance has invalid mesh/material index"; return false; }
    memcpy(sc.camera_view, d->camera_view, sizeof sc.camera_view);
    sc.camera_aspect = d->camera_aspect > 0.0f ? d->camera_aspect : 1.0f;
    return true;
}


// ================================================================================================ Wavefront OBJ / MTL
// The reference imports every format through assimp (AssetImporterImpl.cpp:82-97: Triangulate | GenNormals | GenUVCoords | CalcTangentSpace |
// JoinIdenticalVertices | SortByPType | OptimizeMeshes | OptimizeGraph | FlipUVs) and then reads a fixed set of material keys (:353-455).
// This reader restates that path for OBJ.  PARITY UNPINNED: assimp is not available here and the reference ships no OBJ asset, so the
// importer-specific parts below follow assimp 6.0.2's ObjFileParser / ObjFileMtlImporter from upstream knowledge (SURVEY 8c):
//   geometry   one mesh per (object / group, material) run; polygons -> triangle fans; a face vertex is (v, vt, vn), merged when all three
//              agree (JoinIdenticalVertices); faces without vn get their flat face normal (GenNormals runs on unshared vertices);
//              uv = (u, 1 - v) (FlipUVs); vertices in first-use order; one instance per mesh, Transform = diag(1,-1,1,1) (:233-247)
//   materials  index 0 = assimp's "DefaultMaterial" (Kd 0.6), then the newmtl entries in file order.  Keys the reference reads:
//              COLOR_DIFFUSE <- Kd (0.6), COLOR_EMISSIVE <- Ke (0), COLOR_SPECULAR <- Ks (0), REFRACTI <- Ni (1.0: always set by the importer),
//              ROUGHNESS_FACTOR <- Pr (absent -> 1), METALLIC_FACTOR <- Pm (absent -> 0), ANISOTROPY_FACTOR <- aniso, ANISOTROPY_ROTATION <- anisor
//              (radians -> degrees, :404-414); no transmission / emissive-intensity keys.  Textures: DIFFUSE <- map_Kd, NORMALS <- norm / map_Kn,
//              DIFFUSE_ROUGHNESS <- map_Pr, METALNESS <- map_Pm, EMISSIVE <- map_Ke (map_bump / bump go to HEIGHT, which the reference ignores).
//   camera     none in OBJ: the reference's default lookAt((0,0,5), 0, +Y), aspect 16:9 (PathTracer.cpp:171-178)
namespace {
struct ObjMtl { std::string name; b200pt_material m; TexPaths tp; bool has_pr = false, has_pm = false; };
void obj_default_material(b200pt_material &o) {
    memset(&o, 0, sizeof o);
    for (int k = 0; k < 3; k++) { o.BaseColor[k] = 0.6f; o.SpecularColor[k] = 0.0f; o.MediumColor[k] = 1.0f; }
    o.Metallic = 0.0f; o.Roughness = 1.0f; o.IOR = 1.0f;
}
std::vector<std::string> obj_tokens(const std::string &line) {
    std::vector<std::string> t; size_t i = 0;
    while (i < line.size()) {
        while (i < line.size() && (line[i] == ' ' || line[i] == '\t' || line[i] == '\r')) i++;
        size_t j = i; while (j < line.size() && line[j] != ' ' && line[j] != '\t' && line[j] != '\r') j++;
        if (j > i) t.push_back(line.substr(i, j - i));
        i = j;
    }
    return t;
}
bool obj_lines(const std::string &path, std::vector<std::string> &out) {
    std::vector<uint8_t> d; if (!read_all(path, d)) return false;
    std::string cur;
    for (size_t i = 0; i <= d.size(); i++) {
        const char c = i < d.size() ? (char)d[i] : '\n';
        if (c == '\n') {
            if (!cur.empty() && cur.back() == '\r') cur.pop_back();
            if (!cur.empty() && cur.back() == '\\') { cur.pop_back(); cur.push_back(' '); continue; }   // line continuation
            const size_t h = cur.find('#'); if (h != std::string::npos) cur.erase(h);
            out.push_back(cur); cur.clear();
        } else cur.push_back(c);
    }
    return true;
}
bool load_mtl(const std::string &path, const std::string &base, std::vector<ObjMtl> &mats, std::string &err) {
    std::vector<std::string> lines;
    if (!obj_lines(path, lines)) { err = "cannot read material library " + path; return false; }
    ObjMtl *cur = nullptr;
    auto f3v = [](const std::vector<std::string> &t, float out[3]) { for (int k = 0; k < 3; k++) out[k] = (float)atof(t[(size_t)std::min<size_t>(1 + k, t.size() - 1)].c_str()); };
    for (const std::string &ln : lines) {
        const std::vector<std::string> t = obj_tokens(ln);
        if (t.empty()) continue;
        if (t[0] == "newmtl") { mats.emplace_back(); cur = &mats.back(); obj_default_material(cur->m); cur->name = t.size() > 1 ? t[1] : ""; continue; }
        if (!cur || t.size() < 2) continue;
        const std::string &k = t[0];
        const std::string file = base + "/" + t.back();                     // options (-bm, -o, ...) precede the file name
        if (k == "Kd") f3v(t, cur->m.BaseColor);
        else if (k == "Ke") f3v(t, cur->m.EmissiveColor);
        else if (k == "Ks") f3v(t, cur->m.SpecularColor);
        else if (k == "Ni") cur->m.IOR = (float)atof(t[1].c_str());
        else if (k == "Pr") cur->m.Roughness = (float)atof(t[1].c_str());
        else if (k == "Pm") cur->m.Metallic = (float)atof(t[1].c_str());
        else if (k == "aniso") cur->m.Anisotropy = (float)atof(t[1].c_str());
        else if (k == "anisor") cur->m.AnisotropyRotation = (float)atof(t[1].c_str()) * (180.0f / 3.14159265358979323846f);
        else if (k == "map_Kd") cur->tp.base = file;
        else if (k == "norm" || k == "map_Kn") cur->tp.normal = file;
        else if (k == "map_Pr") cur->tp.rough = file;
        else if (k == "map_Pm") cur->tp.metal = file;
        else if (k == "map_Ke") cur->tp.emissive = file;
    }
    return true;
}
} // namespace

bool load_obj_scene(const std::string &path, HostScene &sc, std::string &err) {
    std::vector<std::string> lines;
    if (!obj_lines(path, lines)) { err = "cannot read " + path; return false; }
    std::string base = path; { size_t k = base.find_last_of("/\\"); base = (k == std::string::npos) ? "." : base.substr(0, k); }
    std::vector<float> P, N, T;                                             // v, vn, vt pools
    std::vector<ObjMtl> mats; { ObjMtl d; d.name = "DefaultMaterial"; obj_default_material(d.m); mats.push_back(d); }
    struct Key { int v, t, n; float gn[3]; bool operator<(const Key &o) const { if (v != o.v) return v < o.v; if (t != o.t) return t < o.t; if (n != o.n) return n < o.n; return memcmp(gn, o.gn, sizeof gn) < 0; } };
    struct Build { std::string name; uint32_t material; std::map<Key, uint32_t> index; HostMesh mesh; };
    std::vector<Build> builds;
    std::string group; uint32_t material = 0; bool need_new = true;
    auto current = [&]() -> Build & {
        if (need_new || builds.empty()) { builds.emplace_back(); builds.back().name = group; builds.back().material = material; builds.back().mesh.name = group; need_new = false; }
        return builds.back();
    };
    for (const std::string &ln : lines) {
        const std::vector<std::string> t = obj_tokens(ln);
        if (t.empty()) continue;
        const std::string &k = t[0];
        if (k == "v" && t.size() >= 4) { for (int c = 1; c <= 3; c++) P.push_back((float)atof(t[(size_t)c].c_str())); }
        else if (k == "vn" && t.size() >= 4) { for (int c = 1; c <= 3; c++) N.push_back((float)atof(t[(size_t)c].c_str())); }
        else if (k == "vt" && t.size() >= 2) { T.push_back((float)atof(t[1].c_str())); T.push_back(t.size() >= 3 ? (float)atof(t[2].c_str()) : 0.0f); }
        else if (k == "o" || k == "g") { group = t.size() > 1 ? t[1] : ""; if (!builds.empty() && !builds.back().mesh.indices.empty()) need_new = true; else if (!builds.empty()) { builds.back().name = group; builds.back().mesh.name = group; } }
        else if (k == "mtllib") { for (size_t i = 1; i < t.size(); i++) if (!load_mtl(base + "/" + t[i], base, mats, err)) return false; }
        else if (k == "usemtl") {
            uint32_t found = 0; for (size_t i = 1; i < mats.size(); i++) if (t.size() > 1 && mats[i].name == t[1]) found = (uint32_t)i;
            if (found != material) { material = found; if (!builds.empty() && !builds.back().mesh.indices.empty()) need_new = true; else if (!builds.empty()) builds.back().material = material; }
        }
        else if (k == "f" && t.size() >= 4) {
            Build &b = current();
            std::vector<Key> fv;
            for (size_t i = 1; i < t.size(); i++) {
                Key key{ 0, 0, 0, { 0, 0, 0 } };
                int part = 0; std::string num;
                const std::string tok = t[i] + "/";
                for (char c : tok) {
                    if (c == '/') { const int val = num.empty() ? 0 : atoi(num.c_str()); if (part == 0) key.v = val; else if (part == 1) key.t = val; else if (part == 2) key.n = val; part++; num.clear(); }
                    else num.push_back(c);
                }
                const int nv = (int)(P.size() / 3), nt = (int)(T.size() / 2), nn = (int)(N.size() / 3);
                if (key.v < 0) key.v = nv + key.v + 1;
                if (key.t < 0) key.t = nt + key.t + 1;
                if (key.n < 0) key.n = nn + key.n + 1;
                if (key.v < 1 || key.v > nv || key.t > nt || key.n > nn) { err = "OBJ face index out of range"; return false; }
                fv.push_back(key);
            }
            for (size_t i = 1; i + 1 < fv.size(); i++) {                  // triangle fan
                Key tri[3] = { fv[0], fv[i], fv[i + 1] };
                if (!tri[0].n || !tri[1].n || !tri[2].n) {                 // GenNormals: flat face normal for vertices that have none
                    const float *a = &P[(size_t)(tri[0].v - 1) * 3], *bb = &P[(size_t)(tri[1].v - 1) * 3], *c = &P[(size_t)(tri[2].v - 1) * 3];
                    const float e1[3] = { bb[0] - a[0], bb[1] - a[1], bb[2] - a[2] }, e2[3] = { c[0] - a[0], c[1] - a[1], c[2] - a[2] };
                    float g[3] = { e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0] };
                    const float len = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
                    if (len > 0.0f) { g[0] /= len; g[1] /= len; g[2] /= len; }
                    for (Key &q : tri) if (!q.n) { q.gn[0] = g[0]; q.gn[1] = g[1]; q.gn[2] = g[2]; }
                }
                for (const Key &q : tri) {
                    auto it = b.index.find(q);
                    uint32_t idx;
                    if (it != b.index.end()) idx = it->second;
                    else {
                        idx = (uint32_t)b.mesh.vertices.size(); b.index[q] = idx;
                        b200pt_vertex v; memset(&v, 0, sizeof v);
                        for (int c = 0; c < 3; c++) v.Position[c] = P[(size_t)(q.v - 1) * 3 + c];
                        float nx, ny, nz;
                        if (q.n) { nx = N[(size_t)(q.n - 1) * 3]; ny = N[(size_t)(q.n - 1) * 3 + 1]; nz = N[(size_t)(q.n - 1) * 3 + 2]; } else { nx = q.gn[0]; ny = q.gn[1]; nz = q.gn[2]; }
                        const float inv = 1.0f / sqrtf(nx * nx + ny * ny + nz * nz);       // glm::normalize (:165)
                        v.Normal[0] = nx * inv; v.Normal[1] = ny * inv; v.Normal[2] = nz * inv;
                        if (q.t) { v.TexCoord[0] = T[(size_t)(q.t - 1) * 2]; v.TexCoord[1] = 1.0f - T[(size_t)(q.t - 1) * 2 + 1]; }   // FlipUVs
                        b.mesh.vertices.push_back(v);
                    }
                    b.mesh.indices.push_back(idx);
                }
            }
        }
    }
    for (auto &b : builds) if (!b.mesh.indices.empty()) {
        b200pt_instance in; M4 flip = m4_identity(); flip.m[1][1] = -1.0f; m4_to_colmajor(flip, in.Transform);
        in.MeshIndex = (uint32_t)sc.meshes.size(); in.MaterialIndex = b.material;
        sc.meshes.push_back(std::move(b.mesh)); sc.instances.push_back(in);
    }
    if (sc.meshes.empty()) { err = "No meshes found in scene"; return false; }
    std::vector<TexPaths> tps;
    for (const ObjMtl &m : mats) { sc.materials.push_back(m.m); sc.material_names.push_back(m.name); tps.push_back(m.tp); }
    if (!build_texture_table(sc, tps, err)) return false;
    M4 v = m4_identity(); v.m[2][3] = -5.0f; m4_to_colmajor(v, sc.camera_view); sc.camera_aspect = 16.0f / 9.0f;   // PathTracer.cpp:171-178
    return true;
}

// AssetImporter::ImportScene (AssetImporterImpl.cpp:82-97): the importer is picked by the file extension
bool load_scene_file(const std::string &path, HostScene &sc, std::string &err) {
    const size_t dot = path.find_last_of('.');
    std::string ext = dot == std::string::npos ? "" : path.substr(dot + 1);
    for (char &c : ext) c = (char)tolower((unsigned char)c);
    if (ext == "obj") return load_obj_scene(path, sc, err);
    if (ext == "gltf" || ext == "glb") return load_gltf_scene(path, sc, err);
    err = "unsupported scene format ." + ext + " (glTF 2.0 .gltf / .glb and Wavefront .obj are implemented)";
    return false;
}

} // namespace b200pt
