"""Shared helpers of the test-suite: build the SAME scene for the CPU oracle and for the product (through the C-ABI)."""
import os
import sys
import functools
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import orc, gltf_ref  # noqa: E402  (test infrastructure)

GOLDEN = os.path.join(ROOT, "tests", "golden")
ASSETS = os.path.join(GOLDEN, "assets")      # shipped files of the reference, whole or sampled (tests/golden/make_golden.py)
BASE_SEED = 0x1234ABCD        # SURVEY 8d


@functools.lru_cache(maxsize=None)
def luts():
    return gltf_ref.load_luts_npz(os.path.join(GOLDEN, "luts.npz"))


@functools.lru_cache(maxsize=None)
def scene_dict(name):
    return gltf_ref.load_scene_npz(os.path.join(GOLDEN, name + ".npz"))


@functools.lru_cache(maxsize=None)
def env_small(w=512, h=256, seed=3):
    """synthetic HDR env (raw rgba, alpha 1) + oracle-built pdf/alias"""
    raw = gltf_ref.synthetic_env(w, h, seed)
    env_pdf, alias, total = orc.build_env_alias(raw)
    return raw, env_pdf, alias


def oracle_scene(name, env=None):
    raw, env_pdf, alias = env if env is not None else env_small()
    return orc.Scene(scene_dict(name), env_pdf, alias, luts())


def camera(name):
    sc = scene_dict(name)
    return orc.camera_from_view(sc["camera_view"], sc["aspect"])


def oracle_config(name, **kw):
    vi, pi = camera(name)
    return orc.default_config(ViewInverse=vi, ProjectionInverse=pi, **kw)


ATMOSPHERE_KEYS = ("EnableAtmosphere", "PlanetPosition", "PlanetRadius", "AtmosphereHeight", "RayleighScatteringCoefficientMultiplier", "MieScatteringCoefficientMultiplier",
                   "OzoneAbsorptionCoefficientMultiplier", "RayleighDensityFalloff", "MieDensityFalloff", "OzoneDensityFalloff", "OzonePeak", "SunColor")
_ORC2PT = {"SampleCount": "SamplesPerFrame", "EnvironmentIntensity": "SkyIntensity", "ScreenSplitCount": "ScreenChunkCount"}


def product_tracer(name, W, H, env=None, device=0, scene=None, **cfg_kw):
    """PathTracer handle (C-ABI) with the same scene / env / LUTs / camera / config as oracle_scene + oracle_config (scene: a scene dict
    to use instead of the fixture `name`)."""
    import vpt_b200 as pt
    raw, env_pdf, alias = env if env is not None else env_small()
    t = pt.PathTracer(device)
    t.set_scene(scene_dict(name) if scene is None else scene)
    t.set_env_map(raw)
    t.set_luts(*luts())
    cfg = pt.default_config()
    atm = {k: cfg_kw.pop(k) for k in list(cfg_kw) if k in ATMOSPHERE_KEYS}        # oracle config names == b200pt_atmosphere names (Enable aside)
    if atm: t.set_atmosphere(**{("Enable" if k == "EnableAtmosphere" else k): v for k, v in atm.items()})
    for k, v in cfg_kw.items():
        if k == "Volumes":                       # homogeneous AABB volumes: list of dicts (oracle.orc.VOLUME_DEFAULTS keys)
            for vi, vol in enumerate(v):
                t.add_volume(**vol)
                if vol.get("Grid") is not None: t.add_density_grid(vi, **vol["Grid"]["source"])   # the same arrays oracle.orc.prepare_density_grid was given
        elif k == "PhaseFunction":
            t.set_phase_function(v)
        else:
            setattr(cfg, _ORC2PT.get(k, k), v)
    t.set_config(cfg)
    t.resize(W, H)
    return t


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.sqrt(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30)))


def write_rgbe(path, rgb):
    """minimal RLE Radiance writer for the decoder test"""
    h, w, _ = rgb.shape
    m = rgb.max(-1); e = np.where(m > 1e-32, np.floor(np.log2(np.maximum(m, 1e-38))) + 1, 0)
    scale = np.where(m > 1e-32, 256.0 / (2.0 ** e), 0)
    out = np.zeros((h, w, 4), np.uint8); out[..., :3] = np.clip(rgb * scale[..., None], 0, 255).astype(np.uint8); out[..., 3] = np.where(m > 1e-32, e + 128, 0)
    with open(path, "wb") as f:
        f.write(b"#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n-Y %d +X %d\n" % (h, w))
        for y in range(h):
            f.write(bytes([2, 2, w >> 8, w & 255]))
            for c in range(4):
                row = out[y, :, c]; i = 0
                while i < w:
                    run = 1
                    while i + run < w and run < 127 and row[i + run] == row[i]: run += 1
                    if run >= 4: f.write(bytes([128 + run, row[i]])); i += run
                    else:
                        j = i
                        while j < w and j - i < 128 and not (j + 3 < w and row[j] == row[j + 1] == row[j + 2] == row[j + 3]): j += 1
                        j = max(j, i + 1); f.write(bytes([j - i]) + bytes(row[i:j])); i = j
    return out


def write_synthetic_gltf(tmp_path):
    """Self-authored glTF (+ .bin + four PNG textures) exercising matrices, TRS nesting, every material extension the reference reads, all
    texture slots and u8 / u16 / u32 indices; returns the .gltf path.  Used by the loader tests and the CLI test."""
    import json
    from PIL import Image
    rng = np.random.default_rng(3)
    pos = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0.5]], np.float32)
    nrm = np.array([[0, 0, 2], [0, 0, 1], [0.1, 0, 1], [0, 0.3, 1]], np.float32)
    uv = rng.random((4, 2)).astype(np.float32)
    i8 = np.array([0, 1, 2, 1, 3, 2], np.uint8); i16 = i8.astype(np.uint16); i32 = i8.astype(np.uint32)
    blob = b""; views = []; accs = []
    def add(arr, comp, typ):
        nonlocal blob
        while len(blob) % 4: blob += b"\0"
        views.append({"buffer": 0, "byteOffset": len(blob), "byteLength": arr.nbytes}); blob += arr.tobytes()
        accs.append({"bufferView": len(views) - 1, "componentType": comp, "count": len(arr), "type": typ}); return len(accs) - 1
    aP, aN, aT = add(pos, 5126, "VEC3"), add(nrm, 5126, "VEC3"), add(uv, 5126, "VEC2")
    a8, a16, a32 = add(i8, 5121, "SCALAR"), add(i16, 5123, "SCALAR"), add(i32, 5125, "SCALAR")
    (tmp_path / "s.bin").write_bytes(blob)
    for n in ("base", "nrm", "mr", "em"):
        Image.fromarray(rng.integers(0, 256, (5, 7, 3), dtype=np.uint8), "RGB").save(tmp_path / f"{n}.png")
    g = {"asset": {"version": "2.0"}, "scene": 0, "scenes": [{"nodes": [0, 3]}],
         "nodes": [{"children": [1, 2], "translation": [1, 2, 3], "rotation": [0.1825742, 0.3651484, 0.5477226, 0.7302967], "scale": [1, 2, 0.5]},
                   {"mesh": 0, "matrix": [1, 0, 0, 0, 0, 0, 1, 0, 0, -1, 0, 0, 0.5, 0.25, -2, 1]},
                   {"camera": 0, "translation": [0, 1, 8], "rotation": [0, 0.0871557, 0, 0.9961947]},
                   {"mesh": 1, "scale": [2, 2, 2]}],
         "cameras": [{"type": "perspective", "perspective": {"aspectRatio": 1.5, "yfov": 0.6, "znear": 0.1}}],
         "meshes": [{"primitives": [{"attributes": {"POSITION": aP, "NORMAL": aN, "TEXCOORD_0": aT}, "indices": a8, "material": 0},
                                    {"attributes": {"POSITION": aP, "NORMAL": aN}, "indices": a16, "material": 1}]},
                    {"primitives": [{"attributes": {"POSITION": aP, "NORMAL": aN, "TEXCOORD_0": aT}, "indices": a32}]}],
         "materials": [{"name": "full", "emissiveFactor": [0.5, 0.25, 1.0], "normalTexture": {"index": 1}, "emissiveTexture": {"index": 3},
                        "pbrMetallicRoughness": {"baseColorFactor": [0.1, 0.2, 0.3, 1], "metallicFactor": 0.25, "roughnessFactor": 0.6, "baseColorTexture": {"index": 0}, "metallicRoughnessTexture": {"index": 2}},
                        "extensions": {"KHR_materials_emissive_strength": {"emissiveStrength": 7.5}, "KHR_materials_ior": {"ior": 1.33}, "KHR_materials_transmission": {"transmissionFactor": 0.75},
                                       "KHR_materials_specular": {"specularColorFactor": [0.9, 0.8, 0.7]}, "KHR_materials_anisotropy": {"anisotropyStrength": 0.4, "anisotropyRotation": 0.5}}},
                       {"name": "defaults"}],
         "textures": [{"source": 0}, {"source": 1}, {"source": 2}, {"source": 3}],
         "images": [{"uri": "base.png"}, {"uri": "nrm.png"}, {"uri": "mr.png"}, {"uri": "em.png"}],
         "accessors": accs, "bufferViews": views, "buffers": [{"uri": "s.bin", "byteLength": len(blob)}]}
    p = str(tmp_path / "s.gltf"); open(p, "w").write(json.dumps(g))
    return p


def write_luts_dir(d):
    """The three energy-compensation tables under the file names PathTracer.cpp:199-201 loads."""
    import os
    os.makedirs(d, exist_ok=True)
    for arr, name in zip(luts(), ("ReflectionLookup.bin", "RefractionLookupHitFromOutside.bin", "RefractionLookupHitFromInside.bin")):
        np.ascontiguousarray(arr, np.float32).tofile(os.path.join(str(d), name))
    return str(d)
