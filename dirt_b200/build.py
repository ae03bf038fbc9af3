"""Builds dirt_b200/libdirt_b200.so from csrc/*.cu with nvcc for sm_90a (in-tree, no torch headers).

Replaces the reference's cmake + TensorFlow-flag build (csrc/CMakeLists.txt:16-59, setup.py:14-25).
"""
import glob
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, 'libdirt_b200.so')
SOURCES = ['api.cu', 'setup.cu', 'raster.cu', 'backward.cu', 'exchange.cu', 'texture.cu', 'lighting.cu', 'normals.cu',
           'deterministic.cu', 'derivatives.cu', 'ibl.cu', 'latlong.cu', 'shadow.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-shared']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    return 'nvcc'


def is_stale():
    if not os.path.exists(SO_PATH):
        return True
    so_time = os.path.getmtime(SO_PATH)
    deps = glob.glob(os.path.join(_HERE, 'csrc', '*')) + [os.path.join(_HERE, '..', 'include', 'dirt_b200.h')]
    return any(os.path.getmtime(p) > so_time for p in deps if os.path.exists(p))


def build(force=False, verbose=False):
    """Compile the library if it is missing or older than its sources.  Returns the .so path."""
    if not force and not is_stale():
        return SO_PATH
    srcs = [os.path.join(_HERE, 'csrc', s) for s in SOURCES]
    extra = os.environ.get('DIRT_NVCC_EXTRA', '').split()   # e.g. -DDIRT_RASTER_MIN_BLOCKS=5 (tuning experiments)
    cmd = [_nvcc()] + NVCC_FLAGS + extra + (['-Xptxas', '-v'] if verbose else []) + ['-o', SO_PATH] + srcs
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + ' '.join(cmd) + '\n' + proc.stdout + proc.stderr)
    if verbose:
        print(proc.stderr)
    return SO_PATH


if __name__ == '__main__':
    print(build(force=True, verbose=True))
