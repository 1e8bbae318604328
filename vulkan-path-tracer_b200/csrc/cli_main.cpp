// cli_main.cpp -- b200pt_render: a headless stand-in for the reference's Editor / Application (PathTracer/Editor.cpp, Application.cpp).
// It drives the C-ABI exactly the way the interactive editor drives PathTracer / PostProcessor:
//   Application.cpp:35-72   make sure the three energy-compensation tables exist (bake them on first use: --bake-luts)
//   Editor.cpp:40-48        SetScene(file) -> ResizeImage(1080 * aspect, 1080) unless --size is given
//   Editor.cpp:83-121       one PathTrace() per UI frame until MaxSamplesAccumulated, with the "samples / time / ETA" read-out of :410-426
//   Editor.cpp:354-408      PostProcessor::SetBloomData / SetTonemappingData, PostProcess()
//   Editor.cpp:815-843      SaveToFile(): RGBA8 PNG named <name>_<spp>spp_<sec>s.png when --out is a directory-less stem (:795)
// plus the two things a batch caller needs and the editor does not have: --checkpoint / --resume (b200pt_save/load_checkpoint).
// Plain C++17 over include/b200pt.h; links only libb200pt.so.  Exit code = the first failing B200PT error code (0 on success).
#include "../../include/b200pt.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

static int fail(b200pt_handle h, const char *what, int32_t code) {
    fprintf(stderr, "b200pt_render: %s failed (%d): %s\n", what, code, h ? b200pt_last_error(h) : "");
    if (h) b200pt_destroy(h);
    return code ? code : 1;
}
#define CALL(x) do { int32_t r_ = (x); if (r_ != B200PT_OK) return fail(h, #x, r_); } while (0)

// --adaptive THRESHOLD[,MIN[,INTERVAL]]: a finite threshold >= 0, MIN >= 2, INTERVAL >= 1 (b200pt_set_adaptive's rules)
static bool parse_adaptive(const char *s, b200pt_adaptive &a) {
    b200pt_default_adaptive(&a);
    a.Enable = 1;
    char *end = nullptr;
    const double t = strtod(s, &end);
    if (end == s || !(t >= 0.0 && t < 1e30)) return false;
    a.Threshold = (float)t;
    for (uint32_t *field : { &a.MinSamples, &a.Interval }) {
        if (*end == 0) break;
        if (*end != ',') return false;
        const char *p = end + 1;
        const long v = strtol(p, &end, 10);
        if (end == p || v < 1 || v > 0x7FFFFFFFL) return false;
        *field = (uint32_t)v;
    }
    return *end == 0 && a.MinSamples >= 2;
}

static void usage() {
    fprintf(stderr,
        "usage: b200pt_render --scene s.gltf --env e.hdr --luts DIR --out image.png [options]\n"
        "  --size W H        image size (default: 1080*aspect x 1080 like the reference)\n"
        "  --spp N           samples to accumulate (default 64)      --depth D   MaxDepth (default 200)\n"
        "  --seed S          base seed (default 0x1234ABCD)          --chunks S  ScreenChunkCount (default 1)\n"
        "  --batch F         dispatches per PathTrace call (default 8)\n"
        "  --exposure E --gamma G --bloom THRESHOLD STRENGTH MIPS FALLOFF      post chain (reference defaults)\n"
        "  --volume x0 y0 z0 x1 y1 z1 density r g b   add a homogeneous AABB volume (repeatable); --volume-g G sets the anisotropy of the last one\n"
        "  --phase 0|1|2     phase function: Henyey-Greenstein, Draine, HG + Draine\n"
        "  --sky AZ ALT      sky / sun rotation in degrees (SetSkyAzimuth / SetSkyAltitude, Editor.cpp sky panel)\n"
        "  --atmosphere      render with the atmosphere (SetEnableAtmosphere(true): sun-disk NEE, Rayleigh / Mie / ozone scattering); --sun-color r g b\n"
        "  --adaptive T[,MIN[,INTERVAL]]  adaptive sampling: stop a pixel once the relative standard error of its mean luminance is <= T\n"
        "                    (checked every INTERVAL frames once it has MIN; defaults 64, 32); --spp stays the cap\n"
        "  --denoise [ITER]  keep per-pixel statistics and write the PNG of the denoised image (ITER a-trous iterations, 0 .. 10, default 5);\n"
        "                    --checkpoint still saves the raw accumulation\n"
        "  --checkpoint FILE save the accumulation when done         --resume FILE  continue from a checkpoint\n"
        "  --preview-every K rewrite the output PNG after every K PathTrace calls (the editor's progressive view, Editor.cpp:83-121)\n"
        "  --bake-luts N     bake missing lookup tables into DIR with N samples per texel first (Application.cpp:35-72)\n"
        "  --animation I --time T   pose the glTF scene at time T of animation I (-1: the rest pose) before rendering (b200pt_pose,\n"
        "                    the tree set_scene builds)\n"
        "  --device K        CUDA device ordinal (default 0)         --quiet\n");
}

int main(int argc, char **argv) {
    std::string scene, env, luts, out, ckpt_out, ckpt_in;
    uint32_t W = 0, H = 0, spp = 64, depth = 200, seed = 0x1234ABCDu, chunks = 1, batch = 8, bake = 0, phase = 0, preview = 0;
    int device = 0, animation = -2; float anim_time = 0.0f; bool quiet = false, atmosphere = false, sky = false; float sky_az = 0.0f, sky_al = 0.0f, sun[3] = { 1.0f, 1.0f, 1.0f };
    b200pt_tonemap tm{ 1.0f, 2.2f }; b200pt_bloom bl{ 2.0f, 1.0f, 10, 5.0f };
    std::vector<b200pt_volume> vols;
    b200pt_adaptive adaptive; b200pt_default_adaptive(&adaptive);
    b200pt_denoise_params dn; b200pt_default_denoise(&dn); bool denoise = false;
    for (int i = 1; i < argc; i++) {
        const std::string a = argv[i];
        auto need = [&](int n) { if (i + n >= argc) { usage(); exit(2); } };
        if (a == "--scene") { need(1); scene = argv[++i]; } else if (a == "--env") { need(1); env = argv[++i]; }
        else if (a == "--luts") { need(1); luts = argv[++i]; } else if (a == "--out") { need(1); out = argv[++i]; }
        else if (a == "--size") { need(2); W = (uint32_t)atoi(argv[++i]); H = (uint32_t)atoi(argv[++i]); }
        else if (a == "--spp") { need(1); spp = (uint32_t)atoi(argv[++i]); } else if (a == "--depth") { need(1); depth = (uint32_t)atoi(argv[++i]); }
        else if (a == "--seed") { need(1); seed = (uint32_t)strtoul(argv[++i], nullptr, 0); } else if (a == "--chunks") { need(1); chunks = (uint32_t)atoi(argv[++i]); }
        else if (a == "--batch") { need(1); batch = (uint32_t)atoi(argv[++i]); }
        else if (a == "--exposure") { need(1); tm.Exposure = (float)atof(argv[++i]); } else if (a == "--gamma") { need(1); tm.Gamma = (float)atof(argv[++i]); }
        else if (a == "--bloom") { need(4); bl.BloomThreshold = (float)atof(argv[++i]); bl.BloomStrength = (float)atof(argv[++i]); bl.MipCount = (uint32_t)atoi(argv[++i]); bl.FalloffRange = (float)atof(argv[++i]); }
        else if (a == "--volume") {
            need(10); b200pt_volume v; b200pt_default_volume(&v);
            for (int k = 0; k < 3; k++) v.CornerMin[k] = (float)atof(argv[++i]);
            for (int k = 0; k < 3; k++) v.CornerMax[k] = (float)atof(argv[++i]);
            v.Density = (float)atof(argv[++i]);
            for (int k = 0; k < 3; k++) v.Color[k] = (float)atof(argv[++i]);
            vols.push_back(v);
        }
        else if (a == "--volume-g") { need(1); if (vols.empty()) { usage(); return 2; } vols.back().Anisotropy = (float)atof(argv[++i]); }
        else if (a == "--phase") { need(1); phase = (uint32_t)atoi(argv[++i]); }
        else if (a == "--sky") { need(2); sky = true; sky_az = (float)atof(argv[++i]); sky_al = (float)atof(argv[++i]); }
        else if (a == "--atmosphere") atmosphere = true;
        else if (a == "--sun-color") { need(3); for (int k = 0; k < 3; k++) sun[k] = (float)atof(argv[++i]); }
        else if (a == "--preview-every") { need(1); preview = (uint32_t)atoi(argv[++i]); }
        else if (a == "--adaptive") { need(1); if (!parse_adaptive(argv[++i], adaptive)) { usage(); return 2; } }
        else if (a == "--denoise") {                                        // optional ITER: the next argument when it is a number
            denoise = true;
            if (i + 1 < argc && argv[i + 1][0] >= '0' && argv[i + 1][0] <= '9') {
                char *end = nullptr; const long v = strtol(argv[++i], &end, 10);
                if (*end != 0 || v < 0 || v > 10) { usage(); return 2; }
                dn.Iterations = (uint32_t)v;
            }
        }
        else if (a == "--checkpoint") { need(1); ckpt_out = argv[++i]; } else if (a == "--resume") { need(1); ckpt_in = argv[++i]; }
        else if (a == "--bake-luts") { need(1); bake = (uint32_t)atoi(argv[++i]); } else if (a == "--device") { need(1); device = atoi(argv[++i]); }
        else if (a == "--animation") { need(1); animation = atoi(argv[++i]); if (animation < -1) { usage(); return 2; } }
        else if (a == "--time") { need(1); anim_time = (float)atof(argv[++i]); }
        else if (a == "--quiet") quiet = true;
        else { usage(); return 2; }
    }
    if (scene.empty() || env.empty() || luts.empty() || out.empty() || !spp || !batch) { usage(); return 2; }

    b200pt_handle h = nullptr;
    { int32_t r = b200pt_create(device, &h); if (r != B200PT_OK) return fail(nullptr, "b200pt_create (no CUDA device / library: the product has no CPU path)", r); }
    if (bake) CALL(b200pt_bake_luts_to_dir(h, luts.c_str(), bake, 1u, 0));
    CALL(b200pt_set_luts_dir(h, luts.c_str()));
    CALL(b200pt_set_env_map_file(h, env.c_str()));
    CALL(b200pt_set_scene_file(h, scene.c_str()));                         // also sizes the image to 1080*aspect x 1080 and installs the scene camera
    if (animation >= -1) CALL(b200pt_pose(h, animation, anim_time, 1));
    if (W && H) CALL(b200pt_resize(h, W, H));
    CALL(b200pt_get_size(h, &W, &H));
    b200pt_config cfg; CALL(b200pt_get_config(h, &cfg));
    cfg.MaxDepth = depth; cfg.ScreenChunkCount = chunks; cfg.MaxSamplesAccumulated = spp;
    if (sky) { cfg.SkyRotationAzimuth = sky_az; cfg.SkyRotationAltitude = sky_al; }
    CALL(b200pt_set_config(h, &cfg));
    if (adaptive.Enable) CALL(b200pt_set_adaptive(h, &adaptive));
    if (denoise) CALL(b200pt_set_track_variance(h, 1));
    if (atmosphere) {
        b200pt_atmosphere atm; CALL(b200pt_get_atmosphere(h, &atm));
        atm.Enable = 1; for (int k = 0; k < 3; k++) atm.SunColor[k] = sun[k];
        CALL(b200pt_set_atmosphere(h, &atm));
    }
    for (const auto &v : vols) CALL(b200pt_add_volume(h, &v));
    if (!vols.empty() || phase) CALL(b200pt_set_phase_function(h, phase));
    if (!ckpt_in.empty()) CALL(b200pt_load_checkpoint(h, ckpt_in.c_str()));
    CALL(b200pt_post_set_tonemap(h, &tm)); CALL(b200pt_post_set_bloom(h, &bl));

    uint32_t acc = 0; CALL(b200pt_samples_accumulated(h, &acc));
    const uint32_t start_acc = acc;
    const auto t0 = std::chrono::steady_clock::now();
    uint32_t calls = 0;
    while (acc < spp) {                                                     // Editor::Draw: PathTrace() until all samples are accumulated (Editor.cpp:116-121)
        int32_t done = 0;
        CALL(b200pt_path_trace(h, batch, seed, &done));
        CALL(b200pt_synchronize(h));
        CALL(b200pt_samples_accumulated(h, &acc));
        if (!quiet) {
            const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            const double rate = (double)(acc - start_acc) * W * H / (s > 0 ? s : 1e-9) / 1e6;
            fprintf(stderr, "\rsamples %u / %u   %.2f s   %.1f Mpaths/s   ETA %.1f s   ", acc, spp, s, rate, acc > start_acc ? s * (spp - acc) / (acc - start_acc) : 0.0);
        }
        if (preview && (++calls % preview) == 0 && acc < spp) {             // what the viewport would show right now: post chain on the running mean
            CALL(b200pt_post_process(h)); CALL(b200pt_save_png(h, out.c_str()));
        }
        if (done) break;
    }
    if (!quiet) fprintf(stderr, "\n");
    if (!ckpt_out.empty()) CALL(b200pt_save_checkpoint(h, ckpt_out.c_str()));
    if (denoise) { CALL(b200pt_denoise(h, &dn, nullptr)); CALL(b200pt_post_process_denoised(h)); }
    else CALL(b200pt_post_process(h));
    CALL(b200pt_save_png(h, out.c_str()));
    b200pt_counters c; CALL(b200pt_get_counters(h, &c));
    uint32_t active = 0; CALL(b200pt_active_pixels(h, &active));
    const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    printf("{\"image\": \"%s\", \"size\": [%u, %u], \"spp\": %u, \"seconds\": %.3f, \"paths\": %llu, \"kernel_launches\": %llu, \"active_pixels\": %u}\n",
           out.c_str(), W, H, acc, s, (unsigned long long)c.paths, (unsigned long long)c.kernel_launches, active);
    b200pt_destroy(h);
    return 0;
}
