"""Variant builds of libdirt_b200 for the GPU tests: the product's sources compiled with other compile-time sizes,
outside the tree, and loaded next to the product library.  Each variant is compiled at most once per test session,
whichever test module asks for it first."""
import os
import subprocess

_LOADED = {}

# The grid caps of the small-grid variant (tests/launch_limits.py restates what each one caps).  None divides the sizes
# the tests run, so that every grid-stride loop ends on a partial round.  Two texture CTAs make a stride of 512 elements,
# which the generic forward's C = 5, 6 and 7 do not divide; seven reduction CTAs divide none of the parameter totals.
SMALL_GRID_CAPS = {'DIRT_TEX_MAX_BLOCKS': 2, 'DIRT_TEX_DET_GRID': 2, 'DIRT_LIGHT_MAX_ITEMS_PER_GRID': 3,
                   'DIRT_LIGHT_REDUCE_MAX_BLOCKS': 7, 'DIRT_NORMALS_MAX_BLOCKS': 3, 'DIRT_DET_MAX_BLOCKS': 3,
                   'DIRT_DERIV_MAX_BLOCKS': 3}


def _variant(tmp_path_factory, name, defines):
    if name not in _LOADED:
        from dirt_b200 import _lib, build
        out = str(tmp_path_factory.mktemp('variant') / ('libdirt_b200_%s.so' % name))
        srcs = [os.path.join(os.path.dirname(build.SO_PATH), 'csrc', s) for s in build.SOURCES]
        cmd = [build._nvcc()] + build.NVCC_FLAGS + ['-D%s=%s' % kv for kv in defines.items()] + ['-o', out] + srcs
        proc = subprocess.run(cmd, capture_output=True, text=True)
        assert proc.returncode == 0, proc.stdout + proc.stderr
        _LOADED[name] = _lib.load(out)
    return _LOADED[name]


def four_slot_library(tmp_path_factory):
    """libdirt_b200 built with DIRT_BWD_SLOTS_C4 = DIRT_BWD_SLOTS_C3 = 4: nearly every backward tile overflows its face
    table and runs tile_generic."""
    return _variant(tmp_path_factory, 'slots4', {'DIRT_BWD_SLOTS_C4': 4, 'DIRT_BWD_SLOTS_C3': 4})


def small_grid_library(tmp_path_factory):
    """libdirt_b200 built with every grid cap of SMALL_GRID_CAPS: a few CTAs (or items per gridDim.y) per launch, so
    that modest inputs run many rounds of each grid-stride loop, the last one partial."""
    return _variant(tmp_path_factory, 'small_grid', SMALL_GRID_CAPS)
