"""ctypes binding of the product's C-ABI (libb200pt.so, include/b200pt.h).

This is only a test/bench harness convenience: the product is the C-ABI library itself.  The class mirrors the
reference's `PathTracer` + `PostProcessor` pair (PathTracer/PathTracer.h:83-183, PathTracer/PostProcessor.h:25-33):
same verbs, same argument meaning.  There is NO fallback: if the CUDA library is missing or no GPU is present,
loading / creating a handle raises.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200PT_LIB") or os.path.join(_HERE, "libb200pt.so")   # B200PT_LIB: A/B a differently built library
_LIB = None

OK = 0
ERR_NOT_IMPLEMENTED = -15001
ERR_NO_SCENE = -15002
ERR_WRONG_ARGUMENTS = -15000
ERR_NO_DEVICE = -15004
ERR_INIT_FAILED = -3


class B200ptError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200pt error {code}: {msg}")
        self.code = code


class Material(C.Structure):
    _fields_ = [("BaseColor", C.c_float * 3), ("EmissiveColor", C.c_float * 3), ("SpecularColor", C.c_float * 3),
                ("MediumColor", C.c_float * 3), ("MediumEmissiveColor", C.c_float * 3),
                ("Metallic", C.c_float), ("Roughness", C.c_float), ("IOR", C.c_float), ("Transmission", C.c_float),
                ("Anisotropy", C.c_float), ("AnisotropyRotation", C.c_float), ("MediumDensity", C.c_float), ("MediumAnisotropy", C.c_float),
                ("BaseColorTextureIndex", C.c_uint32), ("NormalTextureIndex", C.c_uint32), ("RoughnessTextureIndex", C.c_uint32),
                ("MetallicTextureIndex", C.c_uint32), ("EmissiveTextureIndex", C.c_uint32)]


class Mesh(C.Structure):
    _fields_ = [("vertices", C.c_void_p), ("indices", C.c_void_p), ("vertex_count", C.c_uint32), ("index_count", C.c_uint32)]


class Instance(C.Structure):
    _fields_ = [("Transform", C.c_float * 16), ("MeshIndex", C.c_uint32), ("MaterialIndex", C.c_uint32)]


class MeshUpdate(C.Structure):      # b200pt_mesh_update
    _fields_ = [("mesh", C.c_uint32), ("vertex_count", C.c_uint32), ("vertices", C.c_void_p)]


VERTEX_DTYPE = np.dtype([("pos", "<f4", 3), ("nrm", "<f4", 3), ("uv", "<f4", 2)])   # b200pt_vertex, the mesh arrays of load_gltf


class Texture(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("channels", C.c_uint32), ("_pad", C.c_uint32), ("data", C.c_void_p)]


class SceneDesc(C.Structure):
    _fields_ = [("meshes", C.c_void_p), ("mesh_count", C.c_uint32), ("_p0", C.c_uint32),
                ("materials", C.c_void_p), ("material_count", C.c_uint32), ("_p1", C.c_uint32),
                ("textures", C.c_void_p), ("texture_count", C.c_uint32), ("_p2", C.c_uint32),
                ("instances", C.c_void_p), ("instance_count", C.c_uint32), ("_p3", C.c_uint32),
                ("camera_view", C.c_float * 16), ("camera_aspect", C.c_float), ("_p4", C.c_uint32)]


class Config(C.Structure):
    _fields_ = [("SamplesPerFrame", C.c_uint32), ("MaxDepth", C.c_uint32), ("MaxLuminance", C.c_float), ("FocusDistance", C.c_float),
                ("DepthOfFieldStrength", C.c_float), ("SkyRotationAzimuth", C.c_float), ("SkyRotationAltitude", C.c_float),
                ("SkyIntensity", C.c_float), ("EmissiveMeshSamplingPDFBias", C.c_float), ("ScreenChunkCount", C.c_uint32),
                ("EnableSkyMIS", C.c_uint32), ("EnableMeshMIS", C.c_uint32), ("ShowEnvMapDirectly", C.c_uint32),
                ("UseOnlyGeometryNormals", C.c_uint32), ("UseEnergyCompensation", C.c_uint32), ("FurnaceTestMode", C.c_uint32),
                ("MaxSamplesAccumulated", C.c_uint32), ("FramesInFlight", C.c_uint32)]


class Volume(C.Structure):     # b200pt_volume (PathTracer::Volume, PT/PathTracer.h:36-70)
    _fields_ = [("CornerMin", C.c_float * 3), ("CornerMax", C.c_float * 3), ("Position", C.c_float * 3), ("Scale", C.c_float * 3),
                ("Color", C.c_float * 3), ("EmissiveColor", C.c_float * 3), ("TemperatureColor", C.c_float * 3),
                ("Density", C.c_float), ("Anisotropy", C.c_float), ("Alpha", C.c_float), ("DropletSize", C.c_float),
                ("DensityDataIndex", C.c_int32), ("MaxDensityInTheGrid", C.c_float), ("UseBlackbody", C.c_int32), ("HasTemperatureData", C.c_int32),
                ("TemperatureGamma", C.c_float), ("TemperatureScale", C.c_float), ("EmissiveColorGamma", C.c_float),
                ("KelvinMin", C.c_int32), ("KelvinMax", C.c_int32),
                ("ApproximatedScatteringForClouds", C.c_uint32), ("ApproximatedScatteringFalloff", C.c_float), ("GridSharpness", C.c_float)]


class DensityGrid(C.Structure):   # b200pt_density_grid
    _fields_ = [("IndexMin", C.c_int32 * 3), ("Dim", C.c_uint32 * 3), ("Density", C.c_void_p), ("Temperature", C.c_void_p),
                ("TemperatureMin", C.c_float), ("TemperatureMax", C.c_float), ("VoxelSize", C.c_double), ("Translation", C.c_double * 3)]


def make_density_grid(density, index_min=(0, 0, 0), temperature=None, voxel_size=1.0, translation=(0.0, 0.0, 0.0), temperature_range=None):
    """b200pt_density_grid over numpy arrays [z][y][x] (float32); returns (struct, keep-alive tuple)."""
    d = np.ascontiguousarray(density, dtype=np.float32)
    t = None if temperature is None else np.ascontiguousarray(temperature, dtype=np.float32)
    g = DensityGrid()
    for k in range(3): g.IndexMin[k] = int(index_min[k]); g.Dim[k] = d.shape[2 - k]; g.Translation[k] = float(translation[k])
    g.Density = d.ctypes.data; g.Temperature = None if t is None else t.ctypes.data
    g.TemperatureMin, g.TemperatureMax = (0.0, 0.0) if temperature_range is None else temperature_range
    g.VoxelSize = float(voxel_size)
    return g, (d, t)


def prepare_density_grid(density, **kw):
    """b200pt_prepare_density_grid (host only): (values, max_densities[32768], corner_min, corner_max, max_density)"""
    g, keep = make_density_grid(density, **kw)
    vals = np.empty(keep[0].shape, np.float32); maj = np.empty(32768, np.float32); cmin = (C.c_float * 3)(); cmax = (C.c_float * 3)(); mx = C.c_float()
    r = lib().b200pt_prepare_density_grid(C.byref(g), vals.ctypes.data_as(C.c_void_p), maj.ctypes.data_as(C.c_void_p), cmin, cmax, C.byref(mx))
    if r != OK: raise B200ptError(r, "prepare_density_grid")
    return vals, maj, tuple(cmin), tuple(cmax), mx.value


MAX_VOLUMES = 100


class Tonemap(C.Structure):
    _fields_ = [("Exposure", C.c_float), ("Gamma", C.c_float)]


class Bloom(C.Structure):
    _fields_ = [("BloomThreshold", C.c_float), ("BloomStrength", C.c_float), ("MipCount", C.c_uint32), ("FalloffRange", C.c_float)]


class Adaptive(C.Structure):    # b200pt_adaptive: per-pixel adaptive sampling (no reference equivalent)
    _fields_ = [("Enable", C.c_uint32), ("Threshold", C.c_float), ("MinSamples", C.c_uint32), ("Interval", C.c_uint32)]


def default_adaptive(**kw):
    a = Adaptive(); lib().b200pt_default_adaptive(C.byref(a))
    for k, v in kw.items(): setattr(a, k, v)
    return a


class DenoiseParams(C.Structure):    # b200pt_denoise_params: the a-trous denoiser (no reference equivalent)
    _fields_ = [("Iterations", C.c_uint32), ("FeatureSamples", C.c_uint32), ("SigmaLuminance", C.c_float), ("SigmaNormal", C.c_float), ("SigmaDepth", C.c_float)]


def default_denoise(**kw):
    d = DenoiseParams(); lib().b200pt_default_denoise(C.byref(d))
    for k, v in kw.items(): setattr(d, k, v)
    return d


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays", "medium_events", "kernel_launches")] + \
               [(n, C.c_float) for n in ("ms_total", "ms_raygen", "ms_extend", "ms_shade", "ms_connect", "ms_resolve")] + \
               [("waves", C.c_uint32), ("bounces", C.c_uint32)]


def build(force=False):
    """Compile libb200pt.so in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(_HERE, "csrc", f) for f in os.listdir(os.path.join(_HERE, "csrc"))] + [os.path.join(_HERE, "..", "include", "b200pt.h")]
    if force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-j8", "-s"])
    return LIB_PATH


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
        L = C.CDLL(LIB_PATH)
        L.b200pt_version.restype = C.c_char_p
        L.b200pt_last_error.restype = C.c_char_p; L.b200pt_last_error.argtypes = [C.c_void_p]
        L.b200pt_partition_global_row.restype = C.c_uint32; L.b200pt_partition_global_row.argtypes = [C.c_uint32] * 4
        L.b200pt_partition_local_row_count.restype = C.c_uint32; L.b200pt_partition_local_row_count.argtypes = [C.c_uint32] * 4
        L.b200pt_free.argtypes = [C.c_void_p]; L.b200pt_free.restype = None
        sig = {
            "b200pt_create": [C.c_int32, C.POINTER(C.c_void_p)], "b200pt_destroy": [C.c_void_p],
            "b200pt_set_scene_file": [C.c_void_p, C.c_char_p], "b200pt_set_scene_arrays": [C.c_void_p, C.POINTER(SceneDesc)],
            "b200pt_set_env_map_file": [C.c_void_p, C.c_char_p], "b200pt_set_env_map": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p],
            "b200pt_set_luts": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p], "b200pt_set_luts_dir": [C.c_void_p, C.c_char_p],
            "b200pt_default_config": [C.POINTER(Config)], "b200pt_set_config": [C.c_void_p, C.POINTER(Config)], "b200pt_get_config": [C.c_void_p, C.POINTER(Config)],
            "b200pt_material_count": [C.c_void_p, C.POINTER(C.c_uint32)], "b200pt_get_material": [C.c_void_p, C.c_uint32, C.POINTER(Material)],
            "b200pt_set_material": [C.c_void_p, C.c_uint32, C.POINTER(Material)], "b200pt_get_material_name": [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32],
            "b200pt_set_camera": [C.c_void_p, C.c_void_p, C.c_void_p], "b200pt_get_camera": [C.c_void_p, C.c_void_p, C.c_void_p],
            "b200pt_camera_from_view": [C.c_void_p, C.c_float, C.c_void_p, C.c_void_p],
            "b200pt_resize": [C.c_void_p, C.c_uint32, C.c_uint32], "b200pt_get_size": [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)],
            "b200pt_reset": [C.c_void_p], "b200pt_add_volume": [C.c_void_p, C.c_void_p],
            "b200pt_save_checkpoint": [C.c_void_p, C.c_char_p], "b200pt_load_checkpoint": [C.c_void_p, C.c_char_p],
            "b200pt_default_volume": [C.c_void_p], "b200pt_set_volume": [C.c_void_p, C.c_uint32, C.c_void_p], "b200pt_remove_volume": [C.c_void_p, C.c_uint32],
            "b200pt_volume_count": [C.c_void_p, C.POINTER(C.c_uint32)], "b200pt_get_volume": [C.c_void_p, C.c_uint32, C.c_void_p],
            "b200pt_add_density_data_to_volume": [C.c_void_p, C.c_uint32, C.c_char_p], "b200pt_remove_density_data_from_volume": [C.c_void_p, C.c_uint32],
            "b200pt_add_density_grid_to_volume": [C.c_void_p, C.c_uint32, C.c_void_p],
            "b200pt_prepare_density_grid": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
            "b200pt_set_phase_function": [C.c_void_p, C.c_uint32], "b200pt_get_phase_function": [C.c_void_p, C.POINTER(C.c_uint32)],
            "b200pt_set_partition": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32], "b200pt_local_rows": [C.c_void_p, C.POINTER(C.c_uint32)],
            "b200pt_path_trace": [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_int32)], "b200pt_samples_accumulated": [C.c_void_p, C.POINTER(C.c_uint32)],
            "b200pt_synchronize": [C.c_void_p], "b200pt_set_stream": [C.c_void_p, C.c_void_p], "b200pt_set_profiling": [C.c_void_p, C.c_int32], "b200pt_get_hdr": [C.c_void_p, C.c_void_p, C.c_int32], "b200pt_hdr_device_ptr": [C.c_void_p, C.POINTER(C.c_void_p)],
            "b200pt_set_hdr": [C.c_void_p, C.c_void_p, C.c_int32], "b200pt_get_counters": [C.c_void_p, C.POINTER(Counters)],
            "b200pt_post_set_tonemap": [C.c_void_p, C.POINTER(Tonemap)], "b200pt_post_set_bloom": [C.c_void_p, C.POINTER(Bloom)],
            "b200pt_post_process": [C.c_void_p], "b200pt_get_ldr": [C.c_void_p, C.c_void_p, C.c_int32], "b200pt_get_bloom": [C.c_void_p, C.c_void_p],
            "b200pt_bloom_mip_sizes": [C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)], "b200pt_save_png": [C.c_void_p, C.c_char_p],
            "b200pt_volume_walks": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
            "b200pt_trace_closest": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p],
            "b200pt_scene_stats": [C.c_void_p] + [C.POINTER(C.c_uint32)] * 4,
            "b200pt_trace_stats": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p],
            "b200pt_trace_query": [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint32] + [C.c_void_p] * 12,
            "b200pt_shade_query": [C.c_void_p, C.c_int32, C.c_uint32] + [C.c_void_p] * 9,
            "b200pt_miss_query": [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4,
            "b200pt_bounce_query": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)],
            "b200pt_bake_lut": [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p],
            "b200pt_bake_luts_to_dir": [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_int32],
            "b200pt_decode_image_file": [C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_void_p)],
            "b200pt_decode_hdr_file": [C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_void_p)],
            "b200pt_write_png": [C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p],
            "b200pt_build_env_alias": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_float)],
            "b200pt_bvh4_collapse": [C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int32)],
            "b200pt_bvh2_sah_build": [C.c_void_p, C.c_uint32, C.c_float, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.POINTER(C.c_double)],
            "b200pt_bvh2_ploc_build": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.POINTER(C.c_double)],
            "b200pt_bvh2_ploc_build_query": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int32),
                                             C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int32)],
            "b200pt_bvh2_reinsert": [C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_int32, C.c_float, C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.c_void_p],
            "b200pt_bvh2_sah_rebuild": [C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.c_void_p],
            "b200pt_load_gltf": [C.c_char_p, C.POINTER(C.POINTER(SceneDesc))], "b200pt_free_scene": [C.POINTER(SceneDesc)],
            "b200pt_default_adaptive": [C.POINTER(Adaptive)], "b200pt_set_adaptive": [C.c_void_p, C.POINTER(Adaptive)],
            "b200pt_get_adaptive": [C.c_void_p, C.POINTER(Adaptive)], "b200pt_get_pixel_stats": [C.c_void_p, C.c_void_p, C.c_void_p],
            "b200pt_active_pixels": [C.c_void_p, C.POINTER(C.c_uint32)],
            "b200pt_set_track_variance": [C.c_void_p, C.c_int32], "b200pt_get_track_variance": [C.c_void_p, C.POINTER(C.c_int32)],
            "b200pt_default_denoise": [C.POINTER(DenoiseParams)], "b200pt_denoise": [C.c_void_p, C.POINTER(DenoiseParams), C.POINTER(C.c_float)],
            "b200pt_get_denoised": [C.c_void_p, C.c_void_p, C.c_int32],
            "b200pt_get_denoise_inputs": [C.c_void_p, C.POINTER(DenoiseParams), C.c_void_p, C.c_void_p, C.c_void_p],
            "b200pt_denoise_image": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(DenoiseParams), C.c_void_p, C.c_int32],
            "b200pt_post_process_denoised": [C.c_void_p],
            "b200pt_instance_count": [C.c_void_p, C.POINTER(C.c_uint32)], "b200pt_get_instance_transforms": [C.c_void_p, C.c_void_p, C.c_uint32],
            "b200pt_update_instance_transforms": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32],
            "b200pt_mesh_count": [C.c_void_p, C.POINTER(C.c_uint32)], "b200pt_mesh_vertex_count": [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)],
            "b200pt_get_mesh_vertices": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32],
            "b200pt_update_mesh_vertices": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_int32],
            "b200pt_animation_count": [C.c_void_p, C.POINTER(C.c_uint32)],
            "b200pt_get_animation": [C.c_void_p, C.c_uint32, C.c_char_p, C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float)],
            "b200pt_pose": [C.c_void_p, C.c_int32, C.c_float, C.c_int32],
            "b200pt_gltf_animation_info": [C.c_char_p, C.c_int32, C.POINTER(C.c_uint32), C.c_char_p, C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float)],
            "b200pt_gltf_pose_nodes": [C.c_char_p, C.c_int32, C.c_float, C.POINTER(C.c_uint32), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)],
        }
        for name, args in sig.items():
            fn = getattr(L, name); fn.restype = C.c_int32; fn.argtypes = args
        _LIB = L
    return _LIB


class Atmosphere(C.Structure):      # b200pt_atmosphere (include/b200pt.h)
    _fields_ = [("Enable", C.c_uint32), ("PlanetPosition", C.c_float * 3), ("PlanetRadius", C.c_float), ("AtmosphereHeight", C.c_float),
                ("RayleighScatteringCoefficientMultiplier", C.c_float * 3), ("MieScatteringCoefficientMultiplier", C.c_float * 3),
                ("OzoneAbsorptionCoefficientMultiplier", C.c_float * 3), ("RayleighDensityFalloff", C.c_float), ("MieDensityFalloff", C.c_float),
                ("OzoneDensityFalloff", C.c_float), ("OzonePeak", C.c_float), ("SunColor", C.c_float * 3)]


# record offsets of b200pt_shade_query (B200PT_SQ_* in include/b200pt.h; tests/test_shading_queries.py checks that they agree)
SQ = dict(N=0, T=3, B=6, NG=9, INSIDE=12, AX=13, AY=14, ETA=15, PM=16, PD=17, PG=18, BASECOLOR=19, ROUGHNESS=22, V=23, H=26, EMITTED=29,
          SKY_L=32, SKY_LV=35, SKY_EVAL=39, SKY_C=43, LIGHT_L=46, LIGHT_LV=49, LIGHT_EVAL=53, LIGHT_C=57, LIGHT_GID=60, BSDF_L=61, BSDF_EVAL=64,
          VALID=68, SCATTER=69, SAMPLE=72, REFRACTED=76, ENTERED=77, REJECTED=78, USER_L=79, USER_EVAL=82, RNG=86, CLASS=87, POS=88, SKY_W=91,
          LIGHT_W=94, STRIDE=97)
# record offsets of b200pt_miss_query (B200PT_MQ_*)
MQ = dict(RGB=0, PDF=3, STRIDE=4)
# record layouts and flags of b200pt_bounce_query (B200PT_BQ_IN_*, B200PT_BQ_OUT_*, B200PT_BQ_STORE / CARRY)
BQ_IN = dict(ORG=0, PDF=3, DIR=4, RNG=7, THR=8, DFLAGS=11, RAD=12, SLOT=15, MEDIUM=16, MEDIUM_G=20, SAMPLE=21, STRIDE=25)
BQ_OUT = dict(T=0, U=1, V=2, INST=3, PRIM=4, ALIVE=5, NEXT=6, SAMPLE=27, CARRY=31, STRIDE=32)
BQ_STORE, BQ_CARRY = 2, 4


def declared_symbols():
    """Every function name declared in include/b200pt.h."""
    import re
    txt = open(os.path.join(_HERE, "..", "include", "b200pt.h")).read()
    return sorted(set(re.findall(r"\b(b200pt_[a-z0-9_]+)\s*\(", txt)))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def default_config(**kw):
    c = Config(); lib().b200pt_default_config(C.byref(c))
    for k, v in kw.items(): setattr(c, k, v)
    return c


def camera_from_view(view16, aspect):
    view16 = np.ascontiguousarray(view16, np.float32); vi = np.zeros(16, np.float32); pi = np.zeros(16, np.float32)
    r = lib().b200pt_camera_from_view(_p(view16), C.c_float(float(aspect)), _p(vi), _p(pi))
    if r != OK: raise B200ptError(r, "camera_from_view")
    return vi, pi


def partition_rows(H, rank, world, band):
    n = lib().b200pt_partition_local_row_count(H, rank, world, band)
    return np.array([lib().b200pt_partition_global_row(i, rank, world, band) for i in range(n)], dtype=np.int64)


def decode_image(path):
    w, h, p = C.c_uint32(), C.c_uint32(), C.c_void_p()
    r = lib().b200pt_decode_image_file(path.encode(), C.byref(w), C.byref(h), C.byref(p))
    if r != OK: raise B200ptError(r, lib().b200pt_last_error(None).decode(errors="replace"))
    a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(h.value, w.value, 4)).copy()
    lib().b200pt_free(p)
    return a


def decode_hdr(path):
    w, h, p = C.c_uint32(), C.c_uint32(), C.c_void_p()
    r = lib().b200pt_decode_hdr_file(path.encode(), C.byref(w), C.byref(h), C.byref(p))
    if r != OK: raise B200ptError(r, lib().b200pt_last_error(None).decode(errors="replace"))
    a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(h.value, w.value, 4)).copy()
    lib().b200pt_free(p)
    return a


def write_png(path, rgba):
    rgba = np.ascontiguousarray(rgba, np.uint8)
    r = lib().b200pt_write_png(path.encode(), rgba.shape[1], rgba.shape[0], _p(rgba))
    if r != OK: raise B200ptError(r, "write_png")


BVH2_DTYPE = np.dtype([("lo0", "<f4", 3), ("hi0", "<f4", 3), ("lo1", "<f4", 3), ("hi1", "<f4", 3), ("c0", "<i4"), ("c1", "<i4"), ("pad", "<u4", 2)])
BVH4_DTYPE = np.dtype([("lox", "<f4", 4), ("loy", "<f4", 4), ("loz", "<f4", 4), ("hix", "<f4", 4), ("hiy", "<f4", 4), ("hiz", "<f4", 4), ("child", "<i4", 4), ("pad", "<u4", 4)])
BVH4_EMPTY = -(1 << 31)


def bvh4_collapse(nodes2, root2=0):
    """Host BVH2 -> BVH4 collapse (csrc/lbvh.cu: bvh4_collapse_host).  nodes2: BVH2_DTYPE array; returns (BVH4_DTYPE array, depth)."""
    nodes2 = np.ascontiguousarray(nodes2, BVH2_DTYPE)
    out = np.zeros(len(nodes2), BVH4_DTYPE)
    n4, d = C.c_uint32(), C.c_int32()
    r = lib().b200pt_bvh4_collapse(_p(nodes2), len(nodes2), int(root2), _p(out), C.byref(n4), C.byref(d))
    if r != OK: raise B200ptError(r, "bvh4_collapse")
    return out[:n4.value].copy(), d.value


def bvh2_sah_rebuild(nodes2, root2=0):
    """Opt-in binned-SAH rebuild of the inner nodes (csrc/lbvh.cu: bvh2_sah_rebuild_host).  Returns (BVH2_DTYPE array, depth, (sah_before, sah_after))."""
    nodes2 = np.ascontiguousarray(nodes2, BVH2_DTYPE)
    out = np.zeros(len(nodes2), BVH2_DTYPE)
    n, d = C.c_uint32(), C.c_int32(); sah = np.zeros(2, np.float64)
    r = lib().b200pt_bvh2_sah_rebuild(_p(nodes2), len(nodes2), int(root2), _p(out), C.byref(n), C.byref(d), _p(sah))
    if r != OK: raise B200ptError(r, "bvh2_sah_rebuild")
    return out[:n.value].copy(), d.value, (float(sah[0]), float(sah[1]))


def bvh2_sah_build(ref_boxes, trav_cost=1.0):
    """Full binned-SAH build from reference boxes [n, 6] (csrc/lbvh.cu: bvh2_sah_build_host).  Returns (nodes, perm, depth, sah_cost)."""
    rb = np.ascontiguousarray(ref_boxes, np.float32).reshape(-1, 6)
    out = np.zeros(max(len(rb) - 1, 1), BVH2_DTYPE); perm = np.zeros(len(rb), np.uint32)
    n, d, c = C.c_uint32(), C.c_int32(), C.c_double()
    r = lib().b200pt_bvh2_sah_build(_p(rb), len(rb), C.c_float(trav_cost), _p(out), _p(perm), C.byref(n), C.byref(d), C.byref(c))
    if r != OK: raise B200ptError(r, "bvh2_sah_build")
    return out[:n.value].copy(), perm, d.value, c.value


def bvh2_ploc_build(ref_boxes):
    """PLOC build from reference boxes [n, 6] in Morton order (csrc/lbvh.cu: bvh2_ploc_build_host, the host restatement of the GPU builder).
    Returns (nodes, perm, depth, sah_cost); no nodes for n <= 4 or an inverted / NaN box."""
    rb = np.ascontiguousarray(ref_boxes, np.float32).reshape(-1, 6)
    out = np.zeros(max(len(rb) - 1, 1), BVH2_DTYPE); perm = np.zeros(len(rb), np.uint32)
    n, d, c = C.c_uint32(), C.c_int32(), C.c_double()
    r = lib().b200pt_bvh2_ploc_build(_p(rb), len(rb), _p(out), _p(perm), C.byref(n), C.byref(d), C.byref(c))
    if r != OK: raise B200ptError(r, "bvh2_ploc_build")
    return out[:n.value].copy(), perm, d.value, c.value


def bvh2_reinsert(nodes2, root2=0, passes=2, fraction=0.25):
    """Insertion-based refinement (csrc/lbvh.cu: bvh2_reinsert_host).  Returns (BVH2_DTYPE array, depth, (sah_before, sah_after))."""
    nodes2 = np.ascontiguousarray(nodes2, BVH2_DTYPE)
    out = np.zeros(len(nodes2), BVH2_DTYPE)
    n, d = C.c_uint32(), C.c_int32(); sah = np.zeros(2, np.float64)
    r = lib().b200pt_bvh2_reinsert(_p(nodes2), len(nodes2), int(root2), _p(out), int(passes), C.c_float(fraction), C.byref(n), C.byref(d), _p(sah))
    if r != OK: raise B200ptError(r, "bvh2_reinsert")
    return out[:n.value].copy(), d.value, (float(sah[0]), float(sah[1]))


def build_env_alias(rgba):
    rgba = np.ascontiguousarray(rgba, np.float32).copy(); h, w = rgba.shape[:2]
    alias = np.zeros(h * w, dtype=np.dtype([("Alias", "<u4"), ("Importance", "<f4")]))
    s = C.c_float()
    r = lib().b200pt_build_env_alias(_p(rgba), w, h, _p(alias), C.byref(s))
    if r != OK: raise B200ptError(r, "build_env_alias")
    return rgba, alias, s.value


def bloom_mip_sizes(W, H):
    wh = np.zeros(20, np.uint32); n = C.c_uint32()
    lib().b200pt_bloom_mip_sizes(W, H, _p(wh), C.byref(n))
    return [(int(wh[2 * i]), int(wh[2 * i + 1])) for i in range(n.value)]


def load_gltf(path):
    """C++ loader -> python dict in the same shape as oracle.gltf_ref.load_gltf (for loader parity tests)."""
    pd = C.POINTER(SceneDesc)()
    r = lib().b200pt_load_gltf(path.encode(), C.byref(pd))
    if r != OK: raise B200ptError(r, lib().b200pt_last_error(None).decode(errors="replace"))
    d = pd.contents
    vdt = VERTEX_DTYPE
    meshes = []
    ms = C.cast(d.meshes, C.POINTER(Mesh))
    for i in range(d.mesh_count):
        v = np.ctypeslib.as_array(C.cast(ms[i].vertices, C.POINTER(C.c_float)), shape=(ms[i].vertex_count, 8)).copy().view(vdt).reshape(-1)
        ix = np.ctypeslib.as_array(C.cast(ms[i].indices, C.POINTER(C.c_uint32)), shape=(ms[i].index_count,)).copy()
        meshes.append((v, ix))
    mats = np.ctypeslib.as_array(C.cast(d.materials, C.POINTER(C.c_uint8)), shape=(d.material_count * 112,)).copy()
    ts = C.cast(d.textures, C.POINTER(Texture)); textures = []
    for i in range(d.texture_count):
        textures.append(np.ctypeslib.as_array(C.cast(ts[i].data, C.POINTER(C.c_uint8)), shape=(ts[i].height, ts[i].width, ts[i].channels)).copy())
    ins = C.cast(d.instances, C.POINTER(Instance)); instances = []
    for i in range(d.instance_count):
        instances.append((np.array(list(ins[i].Transform), np.float32), int(ins[i].MeshIndex), int(ins[i].MaterialIndex)))
    out = dict(meshes=meshes, materials_bytes=mats, textures=textures, instances=instances,
               camera_view=np.array(list(d.camera_view), np.float32), aspect=np.float32(d.camera_aspect))
    lib().b200pt_free_scene(pd)
    return out


def gltf_animations(path):
    """b200pt_gltf_animation_info (host only): [(name, t0, t1)] of a glTF file's animations"""
    L = lib(); n = C.c_uint32(); out = []
    r = L.b200pt_gltf_animation_info(str(path).encode(), -1, C.byref(n), None, 0, None, None)
    if r != OK: raise B200ptError(r, L.b200pt_last_error(None).decode(errors="replace"))
    for i in range(n.value):
        name = C.create_string_buffer(256); t0, t1 = C.c_float(), C.c_float()
        r = L.b200pt_gltf_animation_info(str(path).encode(), i, C.byref(n), name, 256, C.byref(t0), C.byref(t1))
        if r != OK: raise B200ptError(r, L.b200pt_last_error(None).decode(errors="replace"))
        out.append((name.value.decode(errors="replace"), t0.value, t1.value))
    return out


def gltf_pose_nodes(path, animation, t):
    """b200pt_gltf_pose_nodes (host only): (world [nodes, 16] column-major glTF world matrices, [per-node morph weights as float32 arrays])
    of animation `animation` (-1: rest pose) at time t"""
    L = lib(); n, nw = C.c_uint32(), C.c_uint32(); p = str(path).encode()
    r = L.b200pt_gltf_pose_nodes(p, int(animation), C.c_float(t), C.byref(n), None, None, None, C.byref(nw))
    if r != OK: raise B200ptError(r, L.b200pt_last_error(None).decode(errors="replace"))
    world = np.zeros((n.value, 16), np.float32); counts = np.zeros(n.value, np.uint32); w = np.zeros(max(nw.value, 1), np.float32)
    r = L.b200pt_gltf_pose_nodes(p, int(animation), C.c_float(t), C.byref(n), _p(world), _p(counts), _p(w), C.byref(nw))
    if r != OK: raise B200ptError(r, L.b200pt_last_error(None).decode(errors="replace"))
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return world, [w[offs[i]:offs[i + 1]].copy() for i in range(n.value)]


class PathTracer:
    """One GPU: the reference's PathTracer + PostProcessor behind the C-ABI."""

    def __init__(self, device=0):
        self.L = lib(); self.h = C.c_void_p(); self.device = device
        r = self.L.b200pt_create(device, C.byref(self.h))
        if r != OK: raise B200ptError(r, self.L.b200pt_last_error(None).decode(errors="replace"))
        self._keep = []

    def close(self):
        if self.h: self.L.b200pt_destroy(self.h); self.h = C.c_void_p()

    def __del__(self):
        try: self.close()
        except Exception: pass

    def _ck(self, r):
        if r != OK: raise B200ptError(r, self.L.b200pt_last_error(self.h).decode(errors="replace"))

    # ---- volumes: PathTracer::AddVolume / SetVolume / RemoveVolume / SetPhaseFunction (homogeneous AABB volumes)
    @staticmethod
    def make_volume(**kw):
        v = Volume(); r = lib().b200pt_default_volume(C.byref(v))
        if r != OK: raise B200ptError(r, "default_volume")
        for k, val in kw.items():
            if k == "ApproximatedScattering": k = "ApproximatedScatteringForClouds"
            if k == "Grid": continue                                   # density data: add_density_grid after add_volume (tests/util.py)
            if k in ("CornerMin", "CornerMax", "Position", "Scale", "Color", "EmissiveColor", "TemperatureColor"):
                for j in range(3): getattr(v, k)[j] = float(val[j])
            else: setattr(v, k, val)
        return v

    def add_density_grid(self, idx, density, **kw):
        """AddDensityDataToVolume after the file read: density / temperature as numpy [z][y][x] (see make_density_grid)"""
        g, keep = make_density_grid(density, **kw)
        self._ck(self.L.b200pt_add_density_grid_to_volume(self.h, idx, C.byref(g)))

    def remove_density_data(self, idx): self._ck(self.L.b200pt_remove_density_data_from_volume(self.h, idx))

    def add_volume(self, vol=None, **kw):
        v = vol if vol is not None else self.make_volume(**kw)
        self._ck(self.L.b200pt_add_volume(self.h, C.byref(v)))

    def set_volume(self, idx, vol): self._ck(self.L.b200pt_set_volume(self.h, idx, C.byref(vol)))

    def remove_volume(self, idx): self._ck(self.L.b200pt_remove_volume(self.h, idx))

    def volume_count(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_volume_count(self.h, C.byref(n))); return n.value

    def get_volume(self, idx):
        v = Volume(); self._ck(self.L.b200pt_get_volume(self.h, idx, C.byref(v))); return v

    def set_phase_function(self, pf): self._ck(self.L.b200pt_set_phase_function(self.h, pf))

    def get_phase_function(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_get_phase_function(self.h, C.byref(n))); return n.value

    # ---- PathTracer::SetScene
    def set_scene_file(self, path): self._ck(self.L.b200pt_set_scene_file(self.h, path.encode()))

    def set_scene(self, sc):
        """sc: dict as produced by oracle.gltf_ref.load_gltf / load_scene_npz."""
        keep = []
        meshes = (Mesh * len(sc["meshes"]))()
        for i, (v, idx) in enumerate(sc["meshes"]):
            v = np.ascontiguousarray(v); idx = np.ascontiguousarray(idx, np.uint32); keep += [v, idx]
            meshes[i] = Mesh(v.ctypes.data, idx.ctypes.data, len(v), len(idx))
        mats = np.ascontiguousarray(sc["materials"]); keep.append(mats)
        texs = (Texture * len(sc["textures"]))()
        for i, t in enumerate(sc["textures"]):
            t = np.ascontiguousarray(t, np.uint8); keep.append(t)
            texs[i] = Texture(t.shape[1], t.shape[0], t.shape[2], 0, t.ctypes.data)
        insts = (Instance * len(sc["instances"]))()
        for i, (xf, m, mat) in enumerate(sc["instances"]):
            insts[i].MeshIndex = m; insts[i].MaterialIndex = mat
            for k in range(16): insts[i].Transform[k] = float(xf[k])
        d = SceneDesc()
        d.meshes = C.addressof(meshes); d.mesh_count = len(sc["meshes"])
        d.materials = mats.ctypes.data; d.material_count = len(mats)
        d.textures = C.addressof(texs); d.texture_count = len(sc["textures"])
        d.instances = C.addressof(insts); d.instance_count = len(sc["instances"])
        for k in range(16): d.camera_view[k] = float(sc["camera_view"][k])
        d.camera_aspect = float(sc["aspect"])
        self._ck(self.L.b200pt_set_scene_arrays(self.h, C.byref(d)))

    # ---- TLAS::Update: instance transforms (column-major 4x4, b200pt_instance.Transform) without reloading the scene
    def instance_count(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_instance_count(self.h, C.byref(n))); return n.value

    def get_instance_transforms(self):
        """(n, 16) float32, column-major like the scene dict's instance transforms"""
        out = np.zeros((self.instance_count(), 16), np.float32)
        self._ck(self.L.b200pt_get_instance_transforms(self.h, _p(out), len(out))); return out

    REBUILD_GPU = 2     # B200PT_REBUILD_GPU

    def update_instance_transforms(self, xf, rebuild=False):
        """xf: (n, 16) column-major transforms, one per instance.  rebuild: False / 0 refits the tree in place; "gpu" / REBUILD_GPU (2, the C
        API's B200PT_REBUILD_GPU) builds a new tree on the GPU (PLOC, milliseconds); True / 1 builds the tree set_scene would build (host passes)."""
        xf = np.ascontiguousarray(xf, np.float32).reshape(-1, 16)
        mode = self._rebuild_mode(rebuild)
        self._ck(self.L.b200pt_update_instance_transforms(self.h, _p(xf), len(xf), mode))

    def _rebuild_mode(self, rebuild):
        modes = {"gpu": self.REBUILD_GPU, self.REBUILD_GPU: self.REBUILD_GPU, True: 1, False: 0}   # True == 1, False == 0 as keys
        if isinstance(rebuild, (np.integer, np.bool_)): rebuild = rebuild.item()
        if not isinstance(rebuild, (str, bool, int)) or rebuild not in modes:
            raise ValueError(f"rebuild must be False / 0, True / 1 or 'gpu' / {self.REBUILD_GPU}, not {rebuild!r}")
        return modes[rebuild]

    # ---- mesh vertices (no reference equivalent) without reloading the scene
    def mesh_count(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_mesh_count(self.h, C.byref(n))); return n.value

    def get_mesh_vertices(self, mesh):
        """the vertices of mesh `mesh` as a VERTEX_DTYPE array (pos / nrm / uv, as load_gltf returns them)"""
        n = C.c_uint32(); self._ck(self.L.b200pt_mesh_vertex_count(self.h, int(mesh), C.byref(n)))
        out = np.zeros(n.value, VERTEX_DTYPE)
        self._ck(self.L.b200pt_get_mesh_vertices(self.h, int(mesh), _p(out), n.value)); return out

    def update_mesh_vertices(self, updates, rebuild=False):
        """updates: {mesh index: vertices}, each the mesh's whole vertex array, as a VERTEX_DTYPE array, an (n, 8) float32 array
        (pos, nrm, uv) or a contiguous (n, 8) float32 CUDA tensor on this handle's device.  One call takes host arrays or tensors, not both.
        rebuild: as update_instance_transforms.  Tensors are read on the handle's stream after torch's current stream is synchronised."""
        mode = self._rebuild_mode(rebuild)
        items = list(dict(updates).items())
        if not items: raise ValueError("no mesh update")
        on_dev = [hasattr(v, "data_ptr") for _, v in items]
        if any(on_dev) and not all(on_dev): raise ValueError("one call takes host arrays or CUDA tensors, not both")
        ups = (MeshUpdate * len(items))(); keep = []
        for k, (m, v) in enumerate(items):
            if on_dev[k]:
                import torch
                if (not v.is_cuda or v.device.index != self.device or v.dtype != torch.float32 or v.dim() != 2 or v.shape[1] != 8
                        or not v.is_contiguous()):
                    raise ValueError(f"mesh {m}: a CUDA tensor must be contiguous (n, 8) float32 on device {self.device}")
                ptr, n = v.data_ptr(), v.shape[0]
            else:
                v = np.asarray(v)
                if v.dtype.names is not None:
                    if v.dtype != VERTEX_DTYPE: raise ValueError(f"mesh {m}: structured vertices must have dtype {VERTEX_DTYPE}")
                    v = np.ascontiguousarray(v)
                else:
                    if v.ndim != 2 or v.shape[1] != 8: raise ValueError(f"mesh {m}: vertices must be (n, 8) float32 (pos, nrm, uv)")
                    v = np.ascontiguousarray(v, np.float32)
                keep.append(v); ptr, n = v.ctypes.data, len(v)
            ups[k] = MeshUpdate(int(m), n, ptr)
        if any(on_dev):
            import torch
            torch.cuda.current_stream(self.device).synchronize()
        self._ck(self.L.b200pt_update_mesh_vertices(self.h, C.addressof(ups), len(items), 1 if any(on_dev) else 0, mode))

    # ---- glTF animation (no reference equivalent): node animations, skins and morph targets posed on the GPU
    def animations(self):
        """[(name, t0, t1)] of the loaded glTF scene's animations"""
        n = C.c_uint32(); self._ck(self.L.b200pt_animation_count(self.h, C.byref(n))); out = []
        for i in range(n.value):
            name = C.create_string_buffer(256); t0, t1 = C.c_float(), C.c_float()
            self._ck(self.L.b200pt_get_animation(self.h, i, name, 256, C.byref(t0), C.byref(t1)))
            out.append((name.value.decode(errors="replace"), t0.value, t1.value))
        return out

    def pose(self, animation, t, rebuild=False):
        """b200pt_pose: animation `animation` (-1: the rest pose) at time t; rebuild as update_instance_transforms"""
        mode = self._rebuild_mode(rebuild)
        self._ck(self.L.b200pt_pose(self.h, int(animation), C.c_float(t), mode))

    def bvh2_ploc_build_query(self, ref_boxes):
        """b200pt_bvh2_ploc_build_query: the GPU builder and the GPU BVH4 collapse on reference boxes [n, 6] in the given order.
        Returns (nodes, perm, depth, nodes4, depth4)."""
        rb = np.ascontiguousarray(ref_boxes, np.float32).reshape(-1, 6)
        out = np.zeros(max(len(rb) - 1, 1), BVH2_DTYPE); perm = np.zeros(len(rb), np.uint32); out4 = np.zeros(max(len(rb) - 1, 1), BVH4_DTYPE)
        n, d, n4, d4 = C.c_uint32(), C.c_int32(), C.c_uint32(), C.c_int32()
        self._ck(self.L.b200pt_bvh2_ploc_build_query(self.h, _p(rb), len(rb), _p(out), _p(perm), C.byref(n), C.byref(d), _p(out4), C.byref(n4), C.byref(d4)))
        return out[:n.value].copy(), perm, d.value, out4[:n4.value].copy(), d4.value

    def set_env_map(self, rgba):
        rgba = np.ascontiguousarray(rgba, np.float32)
        self._ck(self.L.b200pt_set_env_map(self.h, rgba.shape[1], rgba.shape[0], _p(rgba)))

    def set_env_map_file(self, path): self._ck(self.L.b200pt_set_env_map_file(self.h, path.encode()))

    def set_luts(self, refl, rout, rin):
        a, b, c = [np.ascontiguousarray(x, np.float32) for x in (refl, rout, rin)]
        self._ck(self.L.b200pt_set_luts(self.h, _p(a), _p(b), _p(c)))

    def set_luts_dir(self, d): self._ck(self.L.b200pt_set_luts_dir(self.h, d.encode()))

    # ---- parameters
    def save_checkpoint(self, path): self._ck(self.L.b200pt_save_checkpoint(self.h, str(path).encode()))

    def load_checkpoint(self, path): self._ck(self.L.b200pt_load_checkpoint(self.h, str(path).encode()))

    def set_config(self, cfg): self._ck(self.L.b200pt_set_config(self.h, C.byref(cfg)))

    def get_config(self):
        c = Config(); self._ck(self.L.b200pt_get_config(self.h, C.byref(c))); return c

    def material_count(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_material_count(self.h, C.byref(n))); return n.value

    def get_material(self, i):
        m = Material(); self._ck(self.L.b200pt_get_material(self.h, i, C.byref(m))); return m

    def set_material(self, i, m): self._ck(self.L.b200pt_set_material(self.h, i, C.byref(m)))

    def get_material_name(self, i):
        b = C.create_string_buffer(256); self._ck(self.L.b200pt_get_material_name(self.h, i, b, 256)); return b.value.decode()

    def set_camera(self, vi, pi):
        vi = np.ascontiguousarray(vi, np.float32); pi = np.ascontiguousarray(pi, np.float32)
        self._ck(self.L.b200pt_set_camera(self.h, _p(vi), _p(pi)))

    def get_camera(self):
        vi = np.zeros(16, np.float32); pi = np.zeros(16, np.float32)
        self._ck(self.L.b200pt_get_camera(self.h, _p(vi), _p(pi))); return vi, pi

    def resize(self, w, h): self._ck(self.L.b200pt_resize(self.h, w, h))

    def size(self):
        w, h = C.c_uint32(), C.c_uint32(); self._ck(self.L.b200pt_get_size(self.h, C.byref(w), C.byref(h))); return w.value, h.value

    def reset(self): self._ck(self.L.b200pt_reset(self.h))

    def set_partition(self, rank, world, band): self._ck(self.L.b200pt_set_partition(self.h, rank, world, band))

    def local_rows(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_local_rows(self.h, C.byref(n))); return n.value

    # ---- hot path
    def path_trace(self, dispatches, base_seed):
        done = C.c_int32(); self._ck(self.L.b200pt_path_trace(self.h, dispatches, base_seed & 0xFFFFFFFF, C.byref(done))); return bool(done.value)

    # ---- adaptive sampling
    def set_adaptive(self, adaptive=None, **kw):
        """b200pt_adaptive fields (Enable, Threshold, MinSamples, Interval); unnamed fields take the defaults"""
        a = adaptive if adaptive is not None else default_adaptive(**kw)
        self._ck(self.L.b200pt_set_adaptive(self.h, C.byref(a)))

    def get_adaptive(self):
        a = Adaptive(); self._ck(self.L.b200pt_get_adaptive(self.h, C.byref(a))); return a

    def pixel_stats(self):
        """(frames accumulated per local pixel [rows, W] uint32, relative standard error of the mean luminance [rows, W] float32)"""
        w, _ = self.size(); rows = self.local_rows()
        counts = np.empty((rows, w), np.uint32); rel = np.empty((rows, w), np.float32)
        self._ck(self.L.b200pt_get_pixel_stats(self.h, _p(counts), _p(rel))); return counts, rel

    def active_pixels(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_active_pixels(self.h, C.byref(n))); return n.value

    # ---- per-pixel statistics and the denoiser
    def set_track_variance(self, enable=True): self._ck(self.L.b200pt_set_track_variance(self.h, 1 if enable else 0))

    def get_track_variance(self):
        v = C.c_int32(); self._ck(self.L.b200pt_get_track_variance(self.h, C.byref(v))); return bool(v.value)

    def denoise(self, params=None, **kw):
        """b200pt_denoise (fields of b200pt_denoise_params; unnamed fields take the defaults); returns the device time in ms"""
        p = params if params is not None else default_denoise(**kw)
        ms = C.c_float(); self._ck(self.L.b200pt_denoise(self.h, C.byref(p), C.byref(ms))); return ms.value

    def get_denoised(self, out=None):
        w, h = self.size()
        if out is None: out = np.empty((h, w, 4), np.float32)
        self._ck(self.L.b200pt_get_denoised(self.h, _p(out), 0)); return out

    def denoise_inputs(self, params=None, **kw):
        """(albedo_cov [rows, W, 4], normal_depth [rows, W, 4], variance [rows, W]) of the local rows"""
        p = params if params is not None else default_denoise(**kw)
        w, _ = self.size(); rows = self.local_rows()
        a = np.empty((rows, w, 4), np.float32); n = np.empty((rows, w, 4), np.float32); v = np.empty((rows, w), np.float32)
        self._ck(self.L.b200pt_get_denoise_inputs(self.h, C.byref(p), _p(a), _p(n), _p(v))); return a, n, v

    def denoise_image(self, color, albedo_cov, normal_depth, variance, params=None, **kw):
        """the filter alone on [H, W, 4] / [H, W] arrays; returns the denoised [H, W, 4] float32 image"""
        p = params if params is not None else default_denoise(**kw)
        c, a, n = (np.ascontiguousarray(x, np.float32) for x in (color, albedo_cov, normal_depth))
        v = np.ascontiguousarray(variance, np.float32)
        h, w = c.shape[:2]
        assert a.shape == n.shape == c.shape == (h, w, 4) and v.shape == (h, w)
        out = np.empty((h, w, 4), np.float32)
        self._ck(self.L.b200pt_denoise_image(self.h, w, h, _p(c), _p(a), _p(n), _p(v), C.byref(p), _p(out), 0)); return out

    def post_process_denoised(self): self._ck(self.L.b200pt_post_process_denoised(self.h))

    def samples_accumulated(self):
        n = C.c_uint32(); self._ck(self.L.b200pt_samples_accumulated(self.h, C.byref(n))); return n.value

    def synchronize(self): self._ck(self.L.b200pt_synchronize(self.h))

    def set_stream(self, cuda_stream_ptr): self._ck(self.L.b200pt_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))

    def set_profiling(self, on): self._ck(self.L.b200pt_set_profiling(self.h, 1 if on else 0))

    def get_hdr(self, out=None):
        w, h = self.size(); rows = self.local_rows()
        if out is None: out = np.empty((rows, w, 4), np.float32)
        self._ck(self.L.b200pt_get_hdr(self.h, _p(out), 0)); return out

    def get_hdr_into_device(self, ptr): self._ck(self.L.b200pt_get_hdr(self.h, C.c_void_p(ptr), 1))

    def set_hdr(self, img):
        img = np.ascontiguousarray(img, np.float32); self._ck(self.L.b200pt_set_hdr(self.h, _p(img), 0))

    def set_hdr_from_device(self, ptr): self._ck(self.L.b200pt_set_hdr(self.h, C.c_void_p(ptr), 1))

    def counters(self):
        c = Counters(); self._ck(self.L.b200pt_get_counters(self.h, C.byref(c)))
        return {n: getattr(c, n) for n, _ in Counters._fields_}

    # ---- PostProcessor
    def set_tonemap(self, exposure=1.0, gamma=2.2): self._ck(self.L.b200pt_post_set_tonemap(self.h, C.byref(Tonemap(exposure, gamma))))

    def set_bloom(self, threshold=2.0, strength=1.0, mips=10, falloff=5.0): self._ck(self.L.b200pt_post_set_bloom(self.h, C.byref(Bloom(threshold, strength, mips, falloff))))

    def get_atmosphere(self):
        a = Atmosphere(); self._ck(self.L.b200pt_get_atmosphere(self.h, C.byref(a))); return a

    def set_atmosphere(self, **kw):
        """fields of b200pt_atmosphere (the reference's twelve atmosphere setters); unnamed fields keep their current value"""
        a = self.get_atmosphere()
        for k, v in kw.items():
            if k in ("PlanetPosition", "RayleighScatteringCoefficientMultiplier", "MieScatteringCoefficientMultiplier", "OzoneAbsorptionCoefficientMultiplier", "SunColor"):
                for i in range(3): getattr(a, k)[i] = float(v[i])
            else: setattr(a, k, v)
        self._ck(self.L.b200pt_set_atmosphere(self.h, C.byref(a)))

    def flush(self): self._ck(self.L.b200pt_flush(self.h))

    def post_process(self): self._ck(self.L.b200pt_post_process(self.h))

    def get_ldr(self, out=None):
        w, h = self.size()
        if out is None: out = np.empty((h, w, 4), np.uint8)
        self._ck(self.L.b200pt_get_ldr(self.h, _p(out), 0)); return out

    def accumulate_rows(self, frame_device_ptr, frame_index, y0, y1):
        self._ck(self.L.b200pt_accumulate_rows(self.h, C.c_void_p(frame_device_ptr), C.c_uint32(frame_index), C.c_uint32(y0), C.c_uint32(y1)))

    def post_input_rows(self, y0, y1):
        a, b = C.c_uint32(), C.c_uint32()
        self._ck(self.L.b200pt_post_input_rows(self.h, C.c_uint32(y0), C.c_uint32(y1), C.byref(a), C.byref(b))); return a.value, b.value

    def post_process_rows(self, y0, y1): self._ck(self.L.b200pt_post_process_rows(self.h, C.c_uint32(y0), C.c_uint32(y1)))

    def get_ldr_rows(self, y0, y1, out=None):
        w, h = self.size()
        if out is None: out = np.empty((y1 - y0, w, 4), np.uint8)
        self._ck(self.L.b200pt_get_ldr_rows(self.h, C.c_uint32(y0), C.c_uint32(y1), _p(out), 0)); return out

    def get_ldr_rows_into_device(self, y0, y1, device_ptr):
        self._ck(self.L.b200pt_get_ldr_rows(self.h, C.c_uint32(y0), C.c_uint32(y1), C.c_void_p(device_ptr), 1))

    def get_bloom(self):
        w, h = self.size(); out = np.empty((h, w, 4), np.float32)
        self._ck(self.L.b200pt_get_bloom(self.h, _p(out))); return out

    def save_png(self, path): self._ck(self.L.b200pt_save_png(self.h, path.encode()))

    # ---- test hooks
    def volume_walks(self, org, dirs, seeds, ray_depth=0.0):
        """(T, scatter distance, scattering volume, sampler state after each walk [n, 2]) for every ray / seed"""
        org = np.ascontiguousarray(org, np.float32); dirs = np.ascontiguousarray(dirs, np.float32); seeds = np.ascontiguousarray(seeds, np.uint32); n = len(org)
        T = np.zeros(n, np.float32); sd = np.zeros(n, np.float32); vol = np.zeros(n, np.int32); rng = np.zeros((n, 2), np.uint32)
        self._ck(self.L.b200pt_volume_walks(self.h, n, _p(org), _p(dirs), _p(seeds), C.c_float(ray_depth), _p(T), _p(sd), _p(vol), _p(rng)))
        return T, sd, vol, rng

    def trace_closest(self, org, dirs, tmin, tmax):
        org = np.ascontiguousarray(org, np.float32); dirs = np.ascontiguousarray(dirs, np.float32); n = len(org)
        t = np.zeros(n, np.float32); prim = np.zeros(n, np.uint32); inst = np.zeros(n, np.uint32); uv = np.zeros((n, 2), np.float32)
        self._ck(self.L.b200pt_trace_closest(self.h, n, _p(org), _p(dirs), C.c_float(tmin), C.c_float(tmax), _p(t), _p(prim), _p(inst), _p(uv)))
        return t, prim, inst, uv

    LUT_SIZES = {0: (64, 64, 32), 1: (128, 128, 32), 2: (128, 128, 32)}   # Application.cpp:41,54,67

    def bake_lut(self, kind, sample_count, seed=0, size=None, slices=0):
        """LookupTableCalculator::CalculateTable on the GPU -> (table[z][y][x] float32, device milliseconds)."""
        sx, sy, sz = size or self.LUT_SIZES[kind]
        out = np.zeros((sz, sy, sx), np.float32); ms = C.c_float(0)
        self._ck(self.L.b200pt_bake_lut(self.h, kind, sx, sy, sz, sample_count, seed, slices, _p(out), C.byref(ms)))
        return out, ms.value

    def bake_luts_to_dir(self, path, sample_count=10_000_000, seed=0, overwrite=False):
        self._ck(self.L.b200pt_bake_luts_to_dir(self.h, str(path).encode(), sample_count, seed, int(overwrite)))

    def trace_stats(self, org, dirs, tmin, tmax):
        org = np.ascontiguousarray(org, np.float32); dirs = np.ascontiguousarray(dirs, np.float32); n = len(org)
        st = np.zeros((n, 2), np.uint32)
        self._ck(self.L.b200pt_trace_stats(self.h, n, _p(org), _p(dirs), C.c_float(tmin), C.c_float(tmax), _p(st)))
        return st

    TRAV_SHAPES = {"shared": 0, "global": 1, "flat": 2, "fixed_origin": 3, "dyn2": 4, "dyn4": 5, "dyn4_spill": 6}   # B200PT_TRAV_*
    QUERY_KINDS = {"closest": 0, "any": 1, "target": 2}                                                            # B200PT_QUERY_*

    def trace_query(self, shape, kind, org, dirs, tmin, tmax, target=None, tmax_test=None, fma=False, stats=True):
        """b200pt_trace_query: per-ray tmin / tmax (scalars broadcast).  Returns a dict: closest -> t, prim, inst, uv; any / target ->
        occluded (bool); stats [n, 3] (nodes visited, triangles tested, refused pushes) from the counting instantiations, or None with
        stats=False (the renderer's own instantiations)."""
        org = np.ascontiguousarray(org, np.float32).reshape(-1, 3); dirs = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3); n = len(org)
        lo = np.ascontiguousarray(np.broadcast_to(np.float32(tmin) if np.isscalar(tmin) else np.asarray(tmin, np.float32), (n,)))
        hi = np.ascontiguousarray(np.broadcast_to(np.float32(tmax) if np.isscalar(tmax) else np.asarray(tmax, np.float32), (n,)))
        k = self.QUERY_KINDS[kind]
        tg = np.ascontiguousarray(np.broadcast_to(np.asarray(0xFFFFFFFF if target is None else target, np.uint32), (n,)))
        tt = np.ascontiguousarray(np.broadcast_to(np.asarray(-1.0 if tmax_test is None else tmax_test, np.float32), (n,)))
        t = np.zeros(n, np.float32); prim = np.zeros(n, np.uint32); inst = np.zeros(n, np.uint32); uv = np.zeros((n, 2), np.float32)
        occ = np.zeros(n, np.uint32); st = np.zeros((n, 3), np.uint32) if stats else None
        self._ck(self.L.b200pt_trace_query(self.h, self.TRAV_SHAPES[shape], k, int(bool(fma)), n, _p(org), _p(dirs), _p(lo), _p(hi), _p(tg), _p(tt),
                                           _p(t), _p(prim), _p(inst), _p(uv), _p(occ), _p(st) if stats else None))
        if k == 0: return dict(t=t, prim=prim, inst=inst, uv=uv, stats=st)
        return dict(occluded=occ.astype(bool), stats=st)

    def shade_query(self, inst, prim, uv, dirs, org, pay_pdf, rng, L=None, force_general=False):
        """b200pt_shade_query: one shading step of k_shade_hit per hit.  Returns [n, B200PT_SQ_STRIDE] float32 records; SQ names the offsets."""
        inst = np.ascontiguousarray(inst, np.uint32).reshape(-1); n = len(inst)
        prim = np.ascontiguousarray(np.broadcast_to(np.asarray(prim, np.uint32), (n,)))
        uv = np.ascontiguousarray(np.broadcast_to(np.asarray(uv, np.float32), (n, 2)))
        dirs = np.ascontiguousarray(np.broadcast_to(np.asarray(dirs, np.float32), (n, 3)))
        org = np.ascontiguousarray(np.broadcast_to(np.asarray(org, np.float32), (n, 3)))
        pay_pdf = np.ascontiguousarray(np.broadcast_to(np.asarray(pay_pdf, np.float32), (n,)))
        rng = np.ascontiguousarray(np.broadcast_to(np.asarray(rng, np.uint32), (n,)))
        Lw = None if L is None else np.ascontiguousarray(np.broadcast_to(np.asarray(L, np.float32), (n, 3)))
        out = np.zeros((n, SQ["STRIDE"]), np.float32)
        self._ck(self.L.b200pt_shade_query(self.h, int(bool(force_general)), n, _p(inst), _p(prim), _p(uv), _p(dirs), _p(org), _p(pay_pdf), _p(rng),
                                           None if Lw is None else _p(Lw), _p(out)))
        return out

    def miss_query(self, dirs, depth, pay_pdf):
        """b200pt_miss_query: the renderer's miss shading per world direction.  Returns [n, B200PT_MQ_STRIDE] float32 records (emitted RGB, env pdf)."""
        dirs = np.ascontiguousarray(dirs, np.float32).reshape(-1, 3); n = len(dirs)
        depth = np.ascontiguousarray(np.broadcast_to(np.asarray(depth, np.uint32), (n,)))
        pay_pdf = np.ascontiguousarray(np.broadcast_to(np.asarray(pay_pdf, np.float32), (n,)))
        out = np.zeros((n, MQ["STRIDE"]), np.float32)
        self._ck(self.L.b200pt_miss_query(self.h, n, _p(dirs), _p(depth), _p(pay_pdf), _p(out)))
        return out

    def bounce_query(self, records, store=False, carry=False):
        """b200pt_bounce_query: one bounce of the renderer for [n, BQ_IN["STRIDE"]] float32 path records (u32 fields as their bits).
        Returns ([n, BQ_OUT["STRIDE"]] float32 records, survivor count)."""
        rec = np.ascontiguousarray(records, np.float32).reshape(-1, BQ_IN["STRIDE"]); n = len(rec)
        out = np.zeros((n, BQ_OUT["STRIDE"]), np.float32)
        m = C.c_uint32()
        self._ck(self.L.b200pt_bounce_query(self.h, n, _p(rec), (BQ_STORE if store else 0) | (BQ_CARRY if carry else 0), _p(out), C.byref(m)))
        return out, m.value

    def scene_stats(self):
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._ck(self.L.b200pt_scene_stats(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return dict(triangles=a.value, bvh_nodes=b.value, emissive_meshes=c.value, textures=d.value)
