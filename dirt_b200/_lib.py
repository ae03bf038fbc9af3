"""ctypes binding of libdirt_b200.so (the C ABI declared in include/dirt_b200.h).

Takes the place of `tf.load_op_library(_lib_path + '/librasterise.so')` in the reference
(dirt/rasterise_ops.py:5-10).  Unlike the reference, a missing library is an error, not a warning:
there is no CPU or eager fallback behind this module.
"""
import ctypes
import os

from . import build as _build

_lib = None

ERR_BAD_SHAPE = -1
ERR_NULL_POINTER = -2
ERR_WORKSPACE_TOO_SMALL = -3
ERR_BAD_CHANNEL_GROUPS = -4
ERR_TOO_MANY_VERTICES = -5
ERR_CUDA = -6
ERR_MISALIGNED = -7
ERR_STALE_WORKSPACE = -8
BWD_SHARED_GEOMETRY = 1
BWD_SKIP_POSITION = 2
BWD_SKIP_COLOUR = 4
TEXTURE_BILINEAR = 0
TEXTURE_NEAREST = 1
LIGHT_DIFFUSE_DIRECTIONAL = 0
LIGHT_SPECULAR_DIRECTIONAL = 1
LIGHT_DIFFUSE_POINT = 2
NORMALS_AVERAGE = 0
NORMALS_PRE_SPLIT = 1


def lib():
    """The loaded library.  Raises RuntimeError when libdirt_b200.so has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get('DIRT_B200_LIB') or _build.SO_PATH   # the override serves A/B timing of prebuilt variants (profiles/kbench.py)
    if not os.path.exists(path):
        raise RuntimeError(
            'dirt_b200: %s is missing; rasterisation is unavailable. Build it with '
            '`python -m dirt_b200.build` (needs nvcc, sm_90a).' % path)
    _lib = load(path)
    return _lib


def load(path):
    """A build of the library at `path` (the product one, or a variant compiled with other DIRT_* switches) with the
    argument and result types of every entry point declared."""
    L = ctypes.CDLL(path)
    vp, i, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    L.dirt_error_string.restype = ctypes.c_char_p
    L.dirt_error_string.argtypes = [i]
    L.dirt_abi_version.restype = i
    L.dirt_last_launch_count.restype = i
    L.dirt_workspace_bytes.restype = sz
    L.dirt_workspace_bytes.argtypes = [i] * 6
    L.dirt_workspace_bytes_min.restype = sz
    L.dirt_workspace_bytes_min.argtypes = [i] * 6
    L.dirt_rasterise_forward.restype = i
    L.dirt_rasterise_forward.argtypes = [vp] * 6 + [i] * 6 + [vp, sz, vp]
    L.dirt_rasterise_backward.restype = i
    L.dirt_rasterise_backward.argtypes = [vp] * 8 + [i] * 6 + [ctypes.POINTER(ctypes.c_int), i, i, vp, sz, vp]
    L.dirt_rasterise_backward_ex.restype = i
    L.dirt_rasterise_backward_ex.argtypes = [vp] * 8 + [i] * 6 + [ctypes.POINTER(ctypes.c_int), i, i, i, vp, sz, vp]
    L.dirt_rasterise_backward_deterministic_bytes.restype = sz
    L.dirt_rasterise_backward_deterministic_bytes.argtypes = [i] * 6
    L.dirt_rasterise_backward_deterministic.restype = i
    L.dirt_rasterise_backward_deterministic.argtypes = ([vp] * 8 + [i] * 6 + [ctypes.POINTER(ctypes.c_int), i, i, i, vp, sz, vp, sz,
                                                        vp])
    L.dirt_rasterise_derivatives.restype = i
    L.dirt_rasterise_derivatives.argtypes = [vp] * 5 + [i] * 9 + [vp, sz, vp]
    L.dirt_workspace_status.restype = i
    L.dirt_workspace_status.argtypes = [vp, sz] + [i] * 6 + [vp]
    L.dirt_rasterise_visibility.restype = i
    L.dirt_rasterise_visibility.argtypes = [vp] * 4 + [i] * 5 + [vp, sz, vp]
    L.dirt_peer_exchange_bytes.restype = sz
    L.dirt_peer_exchange_bytes.argtypes = [i, ctypes.c_longlong]
    L.dirt_peer_exchange.restype = i
    L.dirt_peer_exchange.argtypes = [vp, vp, ctypes.POINTER(vp), ctypes.POINTER(vp), i, i, ctypes.c_longlong, ctypes.c_uint, vp]
    L.dirt_kernel_timer_enable.restype = i
    L.dirt_kernel_timer_enable.argtypes = [i]
    L.dirt_kernel_timer_elapsed_ms.restype = ctypes.c_float
    L.dirt_texture_sample.restype = i
    L.dirt_texture_sample.argtypes = [vp] * 3 + [i] * 5 + [ctypes.c_longlong, i, vp]
    L.dirt_texture_sample_backward.restype = i
    L.dirt_texture_sample_backward.argtypes = [vp] * 5 + [i] * 5 + [ctypes.c_longlong, i, vp]
    L.dirt_texture_sample_backward_deterministic_bytes.restype = sz
    L.dirt_texture_sample_backward_deterministic_bytes.argtypes = [i] * 5 + [ctypes.c_longlong, i]
    L.dirt_texture_sample_backward_deterministic.restype = i
    L.dirt_texture_sample_backward_deterministic.argtypes = [vp] * 5 + [i] * 5 + [ctypes.c_longlong, i, vp, sz, vp]
    L.dirt_texture_mip_levels.restype = i
    L.dirt_texture_mip_levels.argtypes = [i, i]
    L.dirt_texture_mip_pyramid_bytes.restype = sz
    L.dirt_texture_mip_pyramid_bytes.argtypes = [i] * 4
    L.dirt_texture_mip_build.restype = i
    L.dirt_texture_mip_build.argtypes = [vp] * 2 + [i] * 4 + [vp]
    L.dirt_texture_sample_trilinear.restype = i
    L.dirt_texture_sample_trilinear.argtypes = [vp] * 5 + [i] * 5 + [ctypes.c_longlong, vp]
    L.dirt_texture_sample_trilinear_backward_bytes.restype = sz
    L.dirt_texture_sample_trilinear_backward_bytes.argtypes = [i] * 5 + [ctypes.c_longlong, i]
    L.dirt_texture_sample_trilinear_backward.restype = i
    L.dirt_texture_sample_trilinear_backward.argtypes = [vp] * 7 + [i] * 5 + [ctypes.c_longlong, i, vp, sz, vp]
    L.dirt_cubemap_atlas_bytes.restype = sz
    L.dirt_cubemap_atlas_bytes.argtypes = [i] * 3
    L.dirt_cubemap_sample.restype = i
    L.dirt_cubemap_sample.argtypes = [vp] * 4 + [i] * 4 + [ctypes.c_longlong, i, vp]
    L.dirt_cubemap_sample_backward_bytes.restype = sz
    L.dirt_cubemap_sample_backward_bytes.argtypes = [i] * 4 + [ctypes.c_longlong, i, i]
    L.dirt_cubemap_sample_backward.restype = i
    L.dirt_cubemap_sample_backward.argtypes = [vp] * 5 + [i] * 4 + [ctypes.c_longlong, i, i, vp, sz, vp]
    L.dirt_cubemap_mip_atlas_bytes.restype = sz
    L.dirt_cubemap_mip_atlas_bytes.argtypes = [i] * 3
    L.dirt_cubemap_sample_trilinear.restype = i
    L.dirt_cubemap_sample_trilinear.argtypes = [vp] * 5 + [i] * 4 + [ctypes.c_longlong, vp]
    L.dirt_cubemap_sample_trilinear_backward_bytes.restype = sz
    L.dirt_cubemap_sample_trilinear_backward_bytes.argtypes = [i] * 4 + [ctypes.c_longlong, i]
    L.dirt_cubemap_sample_trilinear_backward.restype = i
    L.dirt_cubemap_sample_trilinear_backward.argtypes = [vp] * 7 + [i] * 4 + [ctypes.c_longlong, i, vp, sz, vp]
    L.dirt_cubemap_ggx_atlas_bytes.restype = sz
    L.dirt_cubemap_ggx_atlas_bytes.argtypes = [i] * 3
    L.dirt_cubemap_ggx_prefilter.restype = i
    L.dirt_cubemap_ggx_prefilter.argtypes = [vp] * 2 + [i] * 3 + [vp]
    L.dirt_cubemap_sample_ggx.restype = i
    L.dirt_cubemap_sample_ggx.argtypes = [vp] * 5 + [i] * 4 + [ctypes.c_longlong, vp]
    L.dirt_cubemap_sample_ggx_backward_bytes.restype = sz
    L.dirt_cubemap_sample_ggx_backward_bytes.argtypes = [i] * 4 + [ctypes.c_longlong, i]
    L.dirt_cubemap_sample_ggx_backward.restype = i
    L.dirt_cubemap_sample_ggx_backward.argtypes = [vp] * 7 + [i] * 4 + [ctypes.c_longlong, i, vp, sz, vp]
    L.dirt_ggx_brdf_table.restype = i
    L.dirt_ggx_brdf_table.argtypes = [vp, i, vp]
    L.dirt_cubemap_sh_project_bytes.restype = sz
    L.dirt_cubemap_sh_project_bytes.argtypes = [i] * 3
    L.dirt_cubemap_sh_project.restype = i
    L.dirt_cubemap_sh_project.argtypes = [vp, vp, vp, sz] + [i] * 3 + [vp]
    L.dirt_cubemap_sh_project_backward.restype = i
    L.dirt_cubemap_sh_project_backward.argtypes = [vp, vp, vp, sz] + [i] * 3 + [vp]
    L.dirt_latlong_samples.restype = i
    L.dirt_latlong_samples.argtypes = [i] * 3
    L.dirt_latlong_to_cubemap.restype = i
    L.dirt_latlong_to_cubemap.argtypes = [vp] * 2 + [i] * 5 + [vp]
    L.dirt_latlong_to_cubemap_backward.restype = i
    L.dirt_latlong_to_cubemap_backward.argtypes = [vp] * 2 + [i] * 5 + [vp]
    ll = ctypes.c_longlong
    light_inputs = [i, i, vp, ll, vp, ll, vp, ll] + [vp, i] * 4
    L.dirt_lighting_workspace_bytes.restype = sz
    L.dirt_lighting_workspace_bytes.argtypes = [i, ll, i]
    L.dirt_lighting_forward.restype = i
    L.dirt_lighting_forward.argtypes = light_inputs + [vp, i, ll, i, vp]
    L.dirt_lighting_backward.restype = i
    L.dirt_lighting_backward.argtypes = light_inputs + [vp] * 9 + [sz, i, ll, i, vp]
    ggx_inputs = [i, i, vp, ll, vp, ll, vp, ll, vp, ll] + [vp, i] * 3
    L.dirt_ggx_lighting_forward.restype = i
    L.dirt_ggx_lighting_forward.argtypes = ggx_inputs + [vp, i, ll, i, vp]
    L.dirt_ggx_lighting_backward.restype = i
    L.dirt_ggx_lighting_backward.argtypes = ggx_inputs + [vp] * 9 + [sz, i, ll, i, vp]
    sh_inputs = [vp, ll, vp, ll, vp, i]
    L.dirt_sh_lighting_workspace_bytes.restype = sz
    L.dirt_sh_lighting_workspace_bytes.argtypes = [i, ll, i]
    L.dirt_sh_lighting_forward.restype = i
    L.dirt_sh_lighting_forward.argtypes = sh_inputs + [vp, i, ll, i, vp]
    L.dirt_sh_lighting_backward.restype = i
    L.dirt_sh_lighting_backward.argtypes = sh_inputs + [vp] * 5 + [sz, i, ll, i, vp]
    L.dirt_normals_workspace_bytes.restype = sz
    L.dirt_normals_workspace_bytes.argtypes = [i, ll, ll]
    L.dirt_normals_forward.restype = i
    L.dirt_normals_forward.argtypes = [i, vp, ll, vp, vp, vp, sz, i, ll, ll, vp]
    L.dirt_normals_backward.restype = i
    L.dirt_normals_backward.argtypes = [i, vp, ll, vp, vp, vp, vp, sz, i, ll, ll, vp]
    tangent_inputs = [vp, ll, vp, ll, ll, vp, ll, vp]
    L.dirt_tangents_workspace_bytes.restype = sz
    L.dirt_tangents_workspace_bytes.argtypes = [i, ll, ll]
    L.dirt_tangents_forward.restype = i
    L.dirt_tangents_forward.argtypes = tangent_inputs + [vp, vp, sz, i, ll, ll, vp]
    L.dirt_tangents_backward.restype = i
    L.dirt_tangents_backward.argtypes = tangent_inputs + [vp] * 5 + [sz, i, ll, ll, vp]
    normal_map_inputs = [vp, ll, vp, ll, vp, ll]
    L.dirt_normal_map_forward.restype = i
    L.dirt_normal_map_forward.argtypes = normal_map_inputs + [vp, i, ll, vp]
    L.dirt_normal_map_backward.restype = i
    L.dirt_normal_map_backward.argtypes = normal_map_inputs + [vp] * 4 + [i, ll, vp]
    shadow_inputs = [vp, ll, vp, vp, i, i, i, i, ctypes.c_float, ctypes.c_float]
    L.dirt_shadow_workspace_bytes.restype = sz
    L.dirt_shadow_workspace_bytes.argtypes = [i, ll]
    L.dirt_shadow_forward.restype = i
    L.dirt_shadow_forward.argtypes = shadow_inputs + [vp, i, ll, vp]
    L.dirt_shadow_backward.restype = i
    L.dirt_shadow_backward.argtypes = shadow_inputs + [vp] * 5 + [sz, i, ll, vp]
    L.dirt_shadow_backward_deterministic_bytes.restype = sz
    L.dirt_shadow_backward_deterministic_bytes.argtypes = [i, ll, i, i, i]
    L.dirt_shadow_backward_deterministic.restype = i
    L.dirt_shadow_backward_deterministic.argtypes = shadow_inputs + [vp] * 5 + [sz, vp, sz, i, ll, vp]
    return L


EXPORTED_SYMBOLS = ['dirt_error_string', 'dirt_abi_version', 'dirt_workspace_bytes', 'dirt_workspace_bytes_min', 'dirt_rasterise_forward',
                    'dirt_rasterise_backward', 'dirt_rasterise_backward_ex', 'dirt_workspace_status',
                    'dirt_rasterise_visibility', 'dirt_peer_exchange_bytes', 'dirt_peer_exchange', 'dirt_last_launch_count',
                    'dirt_kernel_timer_enable', 'dirt_kernel_timer_elapsed_ms', 'dirt_texture_sample',
                    'dirt_texture_sample_backward', 'dirt_lighting_workspace_bytes', 'dirt_lighting_forward',
                    'dirt_lighting_backward', 'dirt_normals_workspace_bytes', 'dirt_normals_forward',
                    'dirt_normals_backward', 'dirt_rasterise_backward_deterministic_bytes',
                    'dirt_rasterise_backward_deterministic', 'dirt_texture_sample_backward_deterministic_bytes',
                    'dirt_texture_sample_backward_deterministic', 'dirt_texture_mip_levels',
                    'dirt_texture_mip_pyramid_bytes', 'dirt_texture_mip_build', 'dirt_texture_sample_trilinear',
                    'dirt_texture_sample_trilinear_backward_bytes', 'dirt_texture_sample_trilinear_backward',
                    'dirt_rasterise_derivatives', 'dirt_sh_lighting_workspace_bytes', 'dirt_sh_lighting_forward',
                    'dirt_sh_lighting_backward', 'dirt_ggx_lighting_forward', 'dirt_ggx_lighting_backward',
                    'dirt_cubemap_atlas_bytes', 'dirt_cubemap_sample', 'dirt_cubemap_sample_backward_bytes',
                    'dirt_cubemap_sample_backward', 'dirt_cubemap_mip_atlas_bytes', 'dirt_cubemap_sample_trilinear',
                    'dirt_cubemap_sample_trilinear_backward_bytes', 'dirt_cubemap_sample_trilinear_backward',
                    'dirt_cubemap_ggx_atlas_bytes', 'dirt_cubemap_ggx_prefilter', 'dirt_cubemap_sample_ggx',
                    'dirt_cubemap_sample_ggx_backward_bytes', 'dirt_cubemap_sample_ggx_backward', 'dirt_ggx_brdf_table',
                    'dirt_cubemap_sh_project_bytes', 'dirt_cubemap_sh_project', 'dirt_cubemap_sh_project_backward',
                    'dirt_latlong_samples', 'dirt_latlong_to_cubemap', 'dirt_latlong_to_cubemap_backward',
                    'dirt_tangents_workspace_bytes', 'dirt_tangents_forward', 'dirt_tangents_backward',
                    'dirt_normal_map_forward', 'dirt_normal_map_backward', 'dirt_shadow_workspace_bytes',
                    'dirt_shadow_forward', 'dirt_shadow_backward', 'dirt_shadow_backward_deterministic_bytes',
                    'dirt_shadow_backward_deterministic']


def error_string(code):
    return lib().dirt_error_string(int(code)).decode()


def check(code, what):
    """Map a C-ABI return code onto the exception the reference op would raise."""
    if code == 0:
        return
    msg = '%s: %s' % (what, error_string(code))
    if code in (ERR_BAD_SHAPE, ERR_BAD_CHANNEL_GROUPS, ERR_TOO_MANY_VERTICES, ERR_NULL_POINTER, ERR_MISALIGNED):
        raise ValueError(msg)  # errors::InvalidArgument in the reference
    raise RuntimeError(msg)
