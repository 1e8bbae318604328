"""ctypes binding of the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE ONLY:
importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class OrcMesh(C.Structure):
    _fields_ = [("verts", C.c_void_p), ("indices", C.c_void_p), ("nverts", C.c_uint32), ("nindices", C.c_uint32)]


class OrcTexture(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("channels", C.c_uint32), ("_pad", C.c_uint32), ("data", C.c_void_p)]


class OrcInstance(C.Structure):
    _fields_ = [("transform", C.c_float * 16), ("mesh", C.c_uint32), ("material", C.c_uint32)]


class OrcSceneDesc(C.Structure):
    _fields_ = [("meshes", C.c_void_p), ("nmeshes", C.c_uint32), ("_p0", C.c_uint32),
                ("materials", C.c_void_p), ("nmaterials", C.c_uint32), ("_p1", C.c_uint32),
                ("textures", C.c_void_p), ("ntextures", C.c_uint32), ("_p2", C.c_uint32),
                ("instances", C.c_void_p), ("ninstances", C.c_uint32), ("_p3", C.c_uint32),
                ("env_rgba", C.c_void_p), ("env_alias", C.c_void_p), ("envW", C.c_uint32), ("envH", C.c_uint32),
                ("lut_reflect", C.c_void_p), ("lut_refract_out", C.c_void_p), ("lut_refract_in", C.c_void_p)]


class OrcVolume(C.Structure):
    _fields_ = [("CornerMin", C.c_float * 3), ("CornerMax", C.c_float * 3), ("Color", C.c_float * 3), ("EmissiveColor", C.c_float * 3),
                ("Density", C.c_float), ("Anisotropy", C.c_float), ("Alpha", C.c_float), ("DropletSize", C.c_float),
                ("ApproximatedScattering", C.c_uint32), ("ApproximatedScatteringFalloff", C.c_float), ("TemperatureColor", C.c_float * 3),
                ("DensityDataIndex", C.c_int32), ("MaxDensityInTheGrid", C.c_float), ("UseBlackbody", C.c_int32), ("HasTemperatureData", C.c_int32),
                ("TemperatureGamma", C.c_float), ("TemperatureScale", C.c_float), ("EmissiveColorGamma", C.c_float),
                ("KelvinMin", C.c_int32), ("KelvinMax", C.c_int32), ("GridSharpness", C.c_float)]


class OrcGrid(C.Structure):
    _fields_ = [("Values", C.c_void_p), ("MaxDensities", C.c_void_p), ("IndexMin", C.c_int32 * 3), ("Dim", C.c_uint32 * 3), ("WorldBBox", C.c_double * 6),
                ("InvVoxelSize", C.c_float * 3), ("Translation", C.c_float * 3)]


class OrcConfig(C.Structure):
    _fields_ = [("ViewInverse", C.c_float * 16), ("ProjectionInverse", C.c_float * 16),
                ("SampleCount", C.c_uint32), ("MaxDepth", C.c_uint32),
                ("MaxLuminance", C.c_float), ("FocusDistance", C.c_float), ("DepthOfFieldStrength", C.c_float),
                ("SkyRotationAzimuth", C.c_float), ("SkyRotationAltitude", C.c_float), ("EnvironmentIntensity", C.c_float),
                ("EmissiveMeshSamplingPDFBias", C.c_float), ("ScreenSplitCount", C.c_uint32),
                ("EnableSkyMIS", C.c_uint32), ("EnableMeshMIS", C.c_uint32), ("ShowEnvMapDirectly", C.c_uint32),
                ("UseOnlyGeometryNormals", C.c_uint32), ("UseEnergyCompensation", C.c_uint32), ("FurnaceTestMode", C.c_uint32),
                ("PhaseFunction", C.c_uint32), ("VolumesCount", C.c_uint32), ("Volumes", C.c_void_p),
                ("EnableAtmosphere", C.c_uint32), ("_padA", C.c_uint32),
                ("PlanetPosition", C.c_float * 3), ("PlanetRadius", C.c_float), ("AtmosphereHeight", C.c_float),
                ("RayleighScatteringCoefficientMultiplier", C.c_float * 3), ("MieScatteringCoefficientMultiplier", C.c_float * 3),
                ("OzoneAbsorptionCoefficientMultiplier", C.c_float * 3),
                ("RayleighDensityFalloff", C.c_float), ("MieDensityFalloff", C.c_float), ("OzoneDensityFalloff", C.c_float), ("OzonePeak", C.c_float),
                ("SunColor", C.c_float * 3), ("GridCount", C.c_uint32), ("Grids", C.c_void_p)]


class OrcCounters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("paths", "segments", "surface_hits", "misses", "shadow_rays", "medium_events")]


class OrcPostConfig(C.Structure):
    _fields_ = [("Exposure", C.c_float), ("Gamma", C.c_float), ("BloomThreshold", C.c_float), ("BloomStrength", C.c_float),
                ("FalloffRange", C.c_float), ("MipCount", C.c_uint32)]


_FAST = False


def use_fast_build():
    """bench.py's CPU arm only: time the -O3 -march=native build (oracle/Makefile target `fast`), compiled on this host.  Must be called before
    the first lib() of the process; the parity tests never call it (they need the strict-IEEE, contraction-free build)."""
    global _FAST
    if _LIB is not None and not _FAST: raise RuntimeError("use_fast_build() after the strict oracle library was loaded")
    _FAST = True


def host_cpu_info():
    """What the CPU arm really has: logical CPUs, model name, cgroup v2 CPU quota (the GPU boxes cap a 128-thread host at a few CPUs' worth of time)."""
    info = {"logical_cpus": os.cpu_count() or 1, "model": None, "cgroup_cpu_max": None, "effective_cpus": float(os.cpu_count() or 1)}
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"): info["model"] = line.split(":", 1)[1].strip(); break
    except OSError: pass
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        info["cgroup_cpu_max"] = f"{q} {per}"
        if q != "max": info["effective_cpus"] = min(info["effective_cpus"], float(q) / float(per))
    except (OSError, ValueError): pass
    try: info["affinity_cpus"] = len(os.sched_getaffinity(0)); info["effective_cpus"] = min(info["effective_cpus"], float(info["affinity_cpus"]))
    except (AttributeError, OSError): pass
    return info


def build(force=False):
    if _FAST:                                    # always rebuilt (-march=native must match THIS host), outside the tree (it may be read-only)
        so = os.path.join(tempfile.mkdtemp(prefix="orc_fast_"), "liboracle_fast.so")
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B", "fast", "FAST_OUT=" + so])
        return so
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("pt_oracle.c", "post_oracle.c", "io_oracle.c", "pt_oracle.h", "orc_math.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = build()
        L = C.CDLL(so)
        if _FAST: shutil.rmtree(os.path.dirname(so), ignore_errors=True)     # mapped already: the temporary copy is not needed any more
        L.orc_pcg_hash.restype = C.c_uint32; L.orc_pcg_hash.argtypes = [C.c_uint32]
        L.orc_rng_floats.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_dielectric_fresnel.restype = C.c_float; L.orc_dielectric_fresnel.argtypes = [C.c_float, C.c_float]
        L.orc_aces_fitted.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_bake_reflect_texel.restype = C.c_float; L.orc_bake_reflect_texel.argtypes = [C.c_uint32] * 5
        L.orc_bake_refract_texel.restype = C.c_float; L.orc_bake_refract_texel.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32]
        L.orc_bake_lut_texel.restype = C.c_float; L.orc_bake_lut_texel.argtypes = [C.c_int] + [C.c_uint32] * 8
        L.orc_build_env_alias.restype = C.c_float; L.orc_build_env_alias.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_camera_from_view.argtypes = [C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
        L.orc_default_config.argtypes = [C.POINTER(OrcConfig)]
        L.orc_grid_transmittance.restype = C.c_float; L.orc_grid_transmittance.argtypes = [C.POINTER(OrcConfig), C.c_uint32, C.c_void_p, C.c_void_p, C.c_float]
        L.orc_grid_sample.restype = C.c_float; L.orc_grid_sample.argtypes = [C.POINTER(OrcConfig), C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_blackbody.restype = None; L.orc_blackbody.argtypes = [C.c_float, C.c_void_p]
        L.orc_load_hdr.restype = C.c_void_p; L.orc_load_hdr.argtypes = [C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_scene_create.restype = C.c_void_p; L.orc_scene_create.argtypes = [C.POINTER(OrcSceneDesc)]
        L.orc_scene_destroy.argtypes = [C.c_void_p]
        L.orc_scene_triangle_count.restype = C.c_uint32; L.orc_scene_triangle_count.argtypes = [C.c_void_p]
        L.orc_scene_emissive_count.restype = C.c_uint32; L.orc_scene_emissive_count.argtypes = [C.c_void_p]
        L.orc_scene_world_triangles.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_trace_closest.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_shade_query.argtypes = [C.c_void_p, C.POINTER(OrcConfig), C.c_uint32] + [C.c_void_p] * 9
        L.orc_shade_query.restype = None
        L.orc_miss_query.argtypes = [C.c_void_p, C.POINTER(OrcConfig), C.c_uint32] + [C.c_void_p] * 4
        L.orc_miss_query.restype = None
        L.orc_bounce_query.argtypes = [C.c_void_p, C.POINTER(OrcConfig), C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
        L.orc_bounce_query.restype = None
        L.orc_render.argtypes = [C.c_void_p, C.POINTER(OrcConfig), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                 C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int, C.POINTER(OrcCounters)]
        L.orc_sample_pixel.argtypes = [C.c_void_p, C.POINTER(OrcConfig), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                       C.c_void_p, C.POINTER(C.c_uint32)]
        L.orc_default_post_config.argtypes = [C.POINTER(OrcPostConfig)]
        L.orc_bloom_mip_sizes.restype = C.c_uint32; L.orc_bloom_mip_sizes.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_post_process.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(OrcPostConfig), C.c_void_p, C.c_void_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def pcg_hash(x):
    return int(lib().orc_pcg_hash(C.c_uint32(x & 0xFFFFFFFF)))


def rng_floats(seed, n):
    out = np.empty(n, dtype=np.float32)
    lib().orc_rng_floats(seed & 0xFFFFFFFF, n, _p(out))
    return out


def load_hdr(path):
    w, h = C.c_uint32(0), C.c_uint32(0)
    p = lib().orc_load_hdr(path.encode(), C.byref(w), C.byref(h))
    if not p:
        raise IOError("orc_load_hdr failed: " + path)
    a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(h.value, w.value, 4)).copy()
    lib().orc_free(p)
    return a


def build_env_alias(rgba):
    """rgba: (H,W,4) float32, modified copy returned with alpha=pdf; alias: structured (Alias u4, Importance f4)."""
    rgba = np.ascontiguousarray(rgba, dtype=np.float32).copy()
    h, w = rgba.shape[:2]
    alias = np.zeros(h * w, dtype=np.dtype([("Alias", "<u4"), ("Importance", "<f4")]))
    s = lib().orc_build_env_alias(_p(rgba), w, h, _p(alias))
    return rgba, alias, float(s)


def camera_from_view(view16, aspect):
    view16 = np.ascontiguousarray(view16, dtype=np.float32)
    vi = np.zeros(16, np.float32); pi = np.zeros(16, np.float32)
    lib().orc_camera_from_view(_p(view16), C.c_float(float(aspect)), _p(vi), _p(pi))
    return vi, pi


VOLUME_DEFAULTS = dict(CornerMin=(-1.0, -1.0, -1.0), CornerMax=(1.0, 1.0, 1.0), Position=(0.0, 0.0, 0.0), Scale=(1.0, 1.0, 1.0), Color=(0.8, 0.8, 0.8),
                       EmissiveColor=(0.0, 0.0, 0.0), TemperatureColor=(1.0, 0.5, 0.0), Density=1.0, Anisotropy=0.0, Alpha=1.0, DropletSize=20.0,
                       UseBlackbody=1, TemperatureGamma=1.0, TemperatureScale=1.0, EmissiveColorGamma=1.0, KelvinMin=500, KelvinMax=8000,
                       ApproximatedScattering=0, ApproximatedScatteringFalloff=0.8, GridSharpness=1.0, Grid=None)   # PT/PathTracer.h:36-70


def prepare_density_grid(density, index_min=(0, 0, 0), temperature=None, voxel_size=1.0, translation=(0.0, 0.0, 0.0), temperature_range=None):
    """AddDensityDataToVolume after the file read (PT/PathTracer.cpp:1391-1452) through orc_prepare_density_grid.  density / temperature: float32
    arrays [z][y][x] over the active-voxel bbox whose minimum index coordinate is index_min (tree().getValue at every coordinate of the bbox);
    voxel_size / translation: the grid's (uniform, axis-aligned) index-to-world map.  Returns the dict set_volumes' "Grid" key wants."""
    vals = np.array(density, dtype=np.float32, order="C", copy=True)
    dz, dy, dx = vals.shape
    temp = None if temperature is None else np.ascontiguousarray(temperature, dtype=np.float32)
    if temp is not None: assert temp.shape == vals.shape
    tmin, tmax = (0.0, 0.0) if temp is None else ((float(temp.min()), float(temp.max())) if temperature_range is None else temperature_range)
    imin = (C.c_int32 * 3)(*[int(v) for v in index_min]); dim = (C.c_uint32 * 3)(dx, dy, dz)
    maj = np.zeros(32768, np.float32); cmin = (C.c_float * 3)(); cmax = (C.c_float * 3)(); mx = C.c_float()
    L = lib()
    L.orc_prepare_density_grid.restype = None
    L.orc_prepare_density_grid(imin, dim, vals.ctypes.data_as(C.c_void_p), None if temp is None else temp.ctypes.data_as(C.c_void_p), C.c_float(tmin), C.c_float(tmax),
                               maj.ctypes.data_as(C.c_void_p), cmin, cmax, C.byref(mx))
    vs = float(voxel_size); tr = [float(t) for t in translation]
    wb = [index_min[k] * vs + tr[k] for k in range(3)] + [(index_min[k] + (dx, dy, dz)[k]) * vs + tr[k] for k in range(3)]   # NanoVDB GridStats: [min, max + 1] through the map
    return dict(values=vals, max_densities=maj, index_min=tuple(int(v) for v in index_min), dim=(dx, dy, dz), world_bbox=wb,
                inv_voxel_size=np.float32(1.0 / vs), translation=tuple(np.float32(t) for t in tr), corner_min=tuple(cmin), corner_max=tuple(cmax),
                max_density=mx.value, has_temperature=temp is not None,
                source=dict(density=np.array(density, dtype=np.float32), index_min=tuple(int(v) for v in index_min), temperature=temp, voxel_size=vs,
                            translation=tuple(tr), temperature_range=(tmin, tmax)))


def set_volumes(cfg, volumes):
    """Attach AABB volumes (list of dicts with the VOLUME_DEFAULTS keys) to an OrcConfig; the arrays are kept alive on cfg.  A volume whose "Grid" is a
    prepare_density_grid() result is heterogeneous: its corners, MaxDensityInTheGrid and DensityDataIndex come from the grid (PathTracer.cpp:1408-1420,1512),
    and the world AABB is Position + Corner * Scale in float32 (VolumeGPU's constructor, PT/PathTracer.h:396-397)."""
    arr = (OrcVolume * max(1, len(volumes)))()
    grids = [v["Grid"] for v in volumes if v.get("Grid") is not None]
    garr = (OrcGrid * max(1, len(grids)))()
    gi = 0
    for i, v in enumerate(volumes):
        d = dict(VOLUME_DEFAULTS); d.update(v)
        g = d["Grid"]
        if g is not None: d["CornerMin"], d["CornerMax"] = g["corner_min"], g["corner_max"]
        pos, scl = np.array(d["Position"], np.float32), np.array(d["Scale"], np.float32)
        lo = pos + np.array(d["CornerMin"], np.float32) * scl; hi = pos + np.array(d["CornerMax"], np.float32) * scl
        for j in range(3): arr[i].CornerMin[j] = lo[j]; arr[i].CornerMax[j] = hi[j]
        for k in ("Color", "EmissiveColor", "TemperatureColor"):
            for j in range(3): getattr(arr[i], k)[j] = float(d[k][j])
        for k in ("Density", "Anisotropy", "Alpha", "DropletSize", "ApproximatedScatteringFalloff", "TemperatureGamma", "TemperatureScale", "EmissiveColorGamma", "GridSharpness"):
            setattr(arr[i], k, float(d[k]))
        for k in ("ApproximatedScattering", "UseBlackbody", "KelvinMin", "KelvinMax"): setattr(arr[i], k, int(d[k]))
        arr[i].DensityDataIndex = -1; arr[i].MaxDensityInTheGrid = 0.0; arr[i].HasTemperatureData = 0
        if g is not None:
            G = garr[gi]
            G.Values = g["values"].ctypes.data; G.MaxDensities = g["max_densities"].ctypes.data
            for j in range(3):
                G.IndexMin[j] = g["index_min"][j]; G.Dim[j] = g["dim"][j]; G.InvVoxelSize[j] = g["inv_voxel_size"]; G.Translation[j] = g["translation"][j]
            for j in range(6): G.WorldBBox[j] = g["world_bbox"][j]
            arr[i].DensityDataIndex = gi; arr[i].MaxDensityInTheGrid = g["max_density"]; arr[i].HasTemperatureData = int(g["has_temperature"])
            gi += 1
    cfg._volumes_keepalive = (arr, garr, grids)
    cfg.Volumes = C.cast(arr, C.c_void_p).value if volumes else None
    cfg.VolumesCount = len(volumes)
    cfg.Grids = C.cast(garr, C.c_void_p).value if grids else None
    cfg.GridCount = len(grids)
    return cfg


def volume_walks(cfg, org, dirs, seeds, ray_depth=0.0):
    """orc_volume_walks: (T, scatter distance, scattering volume, sampler state after each walk [n, 2])"""
    org = np.ascontiguousarray(org, np.float32); dirs = np.ascontiguousarray(dirs, np.float32); seeds = np.ascontiguousarray(seeds, np.uint32); n = len(org)
    T = np.zeros(n, np.float32); sd = np.zeros(n, np.float32); vol = np.zeros(n, np.int32); rng = np.zeros((n, 2), np.uint32)
    L = lib(); L.orc_volume_walks.restype = None
    L.orc_volume_walks(C.byref(cfg), C.c_uint32(n), org.ctypes.data_as(C.c_void_p), dirs.ctypes.data_as(C.c_void_p), seeds.ctypes.data_as(C.c_void_p), C.c_float(ray_depth),
                       T.ctypes.data_as(C.c_void_p), sd.ctypes.data_as(C.c_void_p), vol.ctypes.data_as(C.c_void_p), rng.ctypes.data_as(C.c_void_p))
    return T, sd, vol, rng


def default_config(**kw):
    c = OrcConfig()
    lib().orc_default_config(C.byref(c))
    for k, v in kw.items():
        if k in ("ViewInverse", "ProjectionInverse"):
            for i in range(16): getattr(c, k)[i] = float(v[i])
        elif k == "Volumes":
            set_volumes(c, v)
        elif k in ("PlanetPosition", "RayleighScatteringCoefficientMultiplier", "MieScatteringCoefficientMultiplier", "OzoneAbsorptionCoefficientMultiplier", "SunColor"):
            for i in range(3): getattr(c, k)[i] = float(v[i])
        else:
            setattr(c, k, v)
    return c


def default_post_config(**kw):
    c = OrcPostConfig()
    lib().orc_default_post_config(C.byref(c))
    for k, v in kw.items(): setattr(c, k, v)
    return c


class Scene:
    """Keeps every numpy buffer alive for the lifetime of the C scene."""

    def __init__(self, sc, env_rgba, env_alias, luts):
        L = lib()
        self.keep = []
        meshes = (OrcMesh * len(sc["meshes"]))()
        for i, (v, idx) in enumerate(sc["meshes"]):
            v = np.ascontiguousarray(v); idx = np.ascontiguousarray(idx, dtype=np.uint32)
            self.keep += [v, idx]
            meshes[i] = OrcMesh(v.ctypes.data, idx.ctypes.data, len(v), len(idx))
        mats = np.ascontiguousarray(sc["materials"]); self.keep.append(mats)
        texs = (OrcTexture * len(sc["textures"]))()
        for i, t in enumerate(sc["textures"]):
            t = np.ascontiguousarray(t, dtype=np.uint8); self.keep.append(t)
            texs[i] = OrcTexture(t.shape[1], t.shape[0], t.shape[2], 0, t.ctypes.data)
        insts = (OrcInstance * len(sc["instances"]))()
        for i, (xf, m, mat) in enumerate(sc["instances"]):
            insts[i].mesh = m; insts[i].material = mat
            for k in range(16): insts[i].transform[k] = float(xf[k])
        env_rgba = np.ascontiguousarray(env_rgba, dtype=np.float32); env_alias = np.ascontiguousarray(env_alias)
        luts = [np.ascontiguousarray(l, dtype=np.float32) for l in luts]
        self.keep += [meshes, texs, insts, env_rgba, env_alias] + luts
        d = OrcSceneDesc()
        d.meshes = C.addressof(meshes); d.nmeshes = len(sc["meshes"])
        d.materials = mats.ctypes.data; d.nmaterials = len(mats)
        d.textures = C.addressof(texs); d.ntextures = len(sc["textures"])
        d.instances = C.addressof(insts); d.ninstances = len(sc["instances"])
        d.env_rgba = env_rgba.ctypes.data; d.env_alias = env_alias.ctypes.data
        d.envH, d.envW = env_rgba.shape[0], env_rgba.shape[1]
        d.lut_reflect, d.lut_refract_out, d.lut_refract_in = [l.ctypes.data for l in luts]
        self.desc = d
        self.h = L.orc_scene_create(C.byref(d))
        self.ntris = L.orc_scene_triangle_count(self.h)
        self.n_emissive = L.orc_scene_emissive_count(self.h)

    def __del__(self):
        try:
            if self.h: lib().orc_scene_destroy(self.h); self.h = None
        except Exception:
            pass

    def world_triangles(self):
        tri = np.zeros((self.ntris, 9), np.float32); inst = np.zeros(self.ntris, np.uint32); prim = np.zeros(self.ntris, np.uint32)
        lib().orc_scene_world_triangles(self.h, _p(tri), _p(inst), _p(prim))
        return tri, inst, prim

    def trace_closest(self, org, dirs, tmin, tmax, use_bvh=True):
        org = np.ascontiguousarray(org, np.float32); dirs = np.ascontiguousarray(dirs, np.float32)
        n = len(org)
        t = np.zeros(n, np.float32); prim = np.zeros(n, np.uint32); inst = np.zeros(n, np.uint32); uv = np.zeros((n, 2), np.float32)
        lib().orc_trace_closest(self.h, n, _p(org), _p(dirs), C.c_float(tmin), C.c_float(tmax), int(use_bvh), _p(t), _p(prim), _p(inst), _p(uv))
        return t, prim, inst, uv

    def shade_query(self, cfg, inst, prim, uv, dirs, org, pay_pdf, rng, L=None, stride=97):
        """orc_shade_query: [n, stride] float32 records laid out like B200PT_SQ_* (include/b200pt.h)"""
        inst = np.ascontiguousarray(inst, np.uint32).reshape(-1); n = len(inst)
        b = lambda a, dt, sh: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dt), sh))
        prim, uv, dirs, org = b(prim, np.uint32, (n,)), b(uv, np.float32, (n, 2)), b(dirs, np.float32, (n, 3)), b(org, np.float32, (n, 3))
        pay_pdf, rng = b(pay_pdf, np.float32, (n,)), b(rng, np.uint32, (n,))
        Lw = None if L is None else b(L, np.float32, (n, 3))
        out = np.zeros((n, stride), np.float32)
        lib().orc_shade_query(self.h, C.byref(cfg), n, _p(inst), _p(prim), _p(uv), _p(dirs), _p(org), _p(pay_pdf), _p(rng), None if Lw is None else _p(Lw), _p(out))
        return out

    def miss_query(self, cfg, dirs, depth, pay_pdf):
        """orc_miss_query: [n, 4] float32 records laid out like B200PT_MQ_* (emitted RGB, env pdf)"""
        dirs = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3); n = len(dirs)
        depth = np.ascontiguousarray(np.broadcast_to(np.asarray(depth, np.uint32), (n,)))
        pay_pdf = np.ascontiguousarray(np.broadcast_to(np.asarray(pay_pdf, np.float32), (n,)))
        out = np.zeros((n, 4), np.float32)
        lib().orc_miss_query(self.h, C.byref(cfg), n, _p(dirs), _p(depth), _p(pay_pdf), _p(out))
        return out

    def bounce_query(self, cfg, records, store=False, carry=False):
        """orc_bounce_query: one path segment and the slot fold per [n, 25] record laid out like B200PT_BQ_IN_*.  Returns ([n, 32] float32
        records laid out like B200PT_BQ_OUT_*, number alive)."""
        rec = np.ascontiguousarray(records, np.float32).reshape(-1, 25); n = len(rec)
        out = np.zeros((n, 32), np.float32); m = C.c_uint32()
        lib().orc_bounce_query(self.h, C.byref(cfg), n, _p(rec), (2 if store else 0) | (4 if carry else 0), _p(out), C.byref(m))
        return out, m.value

    def render(self, cfg, W, H, nframes, base_seed, frame0=0, image=None, rank=0, world=1, band_rows=1, nthreads=0):
        if image is None: image = np.zeros((H, W, 4), np.float32)
        cnt = OrcCounters()
        lib().orc_render(self.h, C.byref(cfg), W, H, frame0, nframes, base_seed & 0xFFFFFFFF, rank, world, band_rows, _p(image), nthreads, C.byref(cnt))
        return image, {n: getattr(cnt, n) for n, _ in OrcCounters._fields_}

    def sample_pixel(self, cfg, W, H, x, y, seed):
        out = np.zeros(3, np.float32); seg = C.c_uint32(0)
        lib().orc_sample_pixel(self.h, C.byref(cfg), W, H, x, y, seed & 0xFFFFFFFF, _p(out), C.byref(seg))
        return out, seg.value


def bloom_mip_sizes(W, H):
    wh = np.zeros(20, np.uint32)
    n = lib().orc_bloom_mip_sizes(W, H, _p(wh))
    return [(int(wh[2 * i]), int(wh[2 * i + 1])) for i in range(n)]


def post_process(hdr, pcfg=None, want_bloom=False):
    hdr = np.ascontiguousarray(hdr, np.float32)
    H, W = hdr.shape[:2]
    if pcfg is None: pcfg = default_post_config()
    ldr = np.zeros((H, W, 4), np.uint8)
    bloom = np.zeros((H, W, 4), np.float32) if want_bloom else None
    lib().orc_post_process(_p(hdr), W, H, C.byref(pcfg), _p(ldr), _p(bloom) if want_bloom else None, 0)
    return (ldr, bloom) if want_bloom else ldr
