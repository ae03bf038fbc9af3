"""Variant builds of libdirt_b200 for the mipmapped cube-map tests, compiled and cached by tests/variant_builds.py's
_variant (at most once per test session, outside the tree)."""
from variant_builds import _variant


def no_smem_library(tmp_path_factory):
    """libdirt_b200 built with DIRT_CUBE_MIP_SMEM_FLOATS = 0: the mipmapped cube-map backward pass accumulates every
    level in global memory."""
    return _variant(tmp_path_factory, 'cube_mip_no_smem', {'DIRT_CUBE_MIP_SMEM_FLOATS': 0})
