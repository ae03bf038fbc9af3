"""Variant builds of libdirt_b200 for the GPU tests: the product's sources compiled with other compile-time sizes,
outside the tree, and loaded next to the product library.  Each variant is compiled at most once per test session,
whichever test module asks for it first."""
import os
import subprocess

_LOADED = {}


def four_slot_library(tmp_path_factory):
    """libdirt_b200 built with DIRT_BWD_SLOTS_C4 = DIRT_BWD_SLOTS_C3 = 4: nearly every backward tile overflows its face
    table and runs tile_generic."""
    if 'slots4' not in _LOADED:
        from dirt_b200 import _lib, build
        out = str(tmp_path_factory.mktemp('variant') / 'libdirt_b200_slots4.so')
        srcs = [os.path.join(os.path.dirname(build.SO_PATH), 'csrc', s) for s in build.SOURCES]
        cmd = [build._nvcc()] + build.NVCC_FLAGS + ['-DDIRT_BWD_SLOTS_C4=4', '-DDIRT_BWD_SLOTS_C3=4', '-o', out] + srcs
        proc = subprocess.run(cmd, capture_output=True, text=True)
        assert proc.returncode == 0, proc.stdout + proc.stderr
        _LOADED['slots4'] = _lib.load(out)
    return _LOADED['slots4']
