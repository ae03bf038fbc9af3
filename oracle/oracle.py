"""ctypes wrapper around oracle/libdirt_oracle.so (the CPU oracle).

TEST INFRASTRUCTURE ONLY -- see the header of oracle/dirt_oracle.c.  Nothing under
dirt_b200/ may import this module; only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs do.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, 'libdirt_oracle.so')
_SRC = os.path.join(_HERE, 'dirt_oracle.c')
_lib = None


def build(force=False):
    """Compile oracle/dirt_oracle.c -> oracle/libdirt_oracle.so (gcc, -ffp-contract=off)."""
    if not force and os.path.exists(_SO) and os.path.getmtime(_SO) >= os.path.getmtime(_SRC):
        return _SO
    flags = ['-O2', '-fPIC', '-ffp-contract=off', '-fno-fast-math', '-std=c11', '-shared']
    for cc, extra in (('/usr/bin/gcc', ['-fopenmp']), ('gcc', ['-fopenmp']), ('/usr/bin/gcc', []), ('gcc', [])):
        try:
            subprocess.run([cc] + flags + extra + ['-o', _SO, _SRC, '-lm'], check=True, capture_output=True)
            return _SO
        except (subprocess.CalledProcessError, FileNotFoundError):
            continue
    raise RuntimeError('could not compile the oracle with gcc')


def lib(build_if_stale=True):
    """The loaded oracle.  build_if_stale=False never compiles: a missing library is an error (bench.py, whose tree may
    be read-only, loads what __graft_entry__.build() left)."""
    global _lib
    if _lib is None:
        if build_if_stale:
            build()
        elif not os.path.exists(_SO):
            raise RuntimeError('%s is missing: build it with __graft_entry__.build() or oracle.build()' % _SO)
        _lib = ctypes.CDLL(_SO)
        _lib.dirt_oracle_threads.restype = ctypes.c_int
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def threads():
    return int(lib().dirt_oracle_threads())


def set_threads(n):
    lib().dirt_oracle_set_threads(ctypes.c_int(int(n)))


def default_groups(channels):
    """The reference's greedy channel split, dirt/rasterise_ops.py:80-108."""
    if channels in (1, 3):
        return [channels]
    groups, begin = [], 0
    while begin < channels:
        width = 3 if begin + 3 <= channels else 1
        groups.append(width)
        begin += width
    return groups


def visibility(vertices, faces, height, width):
    """-> face_ids int32 [B,H,W] (-1 background), gbuffer float32 [B,H,W,4]."""
    vertices, faces = _f32(vertices), _i32(faces)
    B, V, _ = vertices.shape
    F = faces.shape[1]
    ids = np.empty((B, height, width), np.int32)
    gbuf = np.empty((B, height, width, 4), np.float32)
    rc = lib().dirt_oracle_visibility(_ptr(vertices), _ptr(faces), _ptr(ids), _ptr(gbuf),
                                      B, height, width, V, F)
    if rc != 0:
        raise RuntimeError('dirt_oracle_visibility failed: %d' % rc)
    return ids, gbuf


def forward(background, vertices, vertex_colors, faces, return_face_ids=False):
    """Batched forward: background [B,H,W,C], vertices [B,V,4], vertex_colors [B,V,C], faces [B,F,3]."""
    background, vertices = _f32(background), _f32(vertices)
    vertex_colors, faces = _f32(vertex_colors), _i32(faces)
    B, H, W, C = background.shape
    V, F = vertices.shape[1], faces.shape[1]
    assert vertices.shape == (B, V, 4) and vertex_colors.shape == (B, V, C) and faces.shape == (B, F, 3)
    pixels = np.empty_like(background)
    ids = np.empty((B, H, W), np.int32)
    rc = lib().dirt_oracle_forward(_ptr(background), _ptr(vertices), _ptr(vertex_colors), _ptr(faces),
                                   _ptr(pixels), _ptr(ids), B, H, W, C, V, F)
    if rc != 0:
        raise RuntimeError('dirt_oracle_forward failed: %d' % rc)
    return (pixels, ids) if return_face_ids else pixels


def backward(vertices, faces, pixels, grad_pixels, channel_groups=None, return_dilation=False):
    """RasteriseGrad: -> grad_background [B,H,W,C], grad_vertices [B,V,4], grad_vertex_colors [B,V,C].
    With return_dilation, also a list with one bool [B,H,W] mask per channel group (the given groups, or the greedy
    split): the pixels whose position gradient goes to a neighbour's face, as oracle/ref.py backward returns them from
    the reference kernel.  With return_dilation='codes' the list holds uint8 [B,H,W] planes of the full dilation codes
    instead, as dirt_rasterise_backward_deterministic leaves them in its scratch (include/dirt_b200.h): bits 0-1 none /
    own face / first / second neighbour, bit 2 the step along the row; the mask is (code & 3) >= 2."""
    vertices, faces = _f32(vertices), _i32(faces)
    pixels, grad_pixels = _f32(pixels), _f32(grad_pixels)
    B, H, W, C = pixels.shape
    V, F = vertices.shape[1], faces.shape[1]
    assert grad_pixels.shape == pixels.shape
    gb = np.empty_like(pixels)
    gv = np.empty((B, V, 4), np.float32)
    gc = np.empty((B, V, C), np.float32)
    if channel_groups is None:
        groups_ptr, ng = None, 0
    else:
        arr = (ctypes.c_int * len(channel_groups))(*channel_groups)
        groups_ptr, ng = arr, len(channel_groups)
    n_masks = len(channel_groups) if channel_groups is not None else len(default_groups(C))
    dilated = np.zeros((n_masks, B, H, W), np.uint8) if return_dilation else None   # codes (see above)
    rc = lib().dirt_oracle_backward_ex(_ptr(vertices), _ptr(faces), _ptr(pixels), _ptr(grad_pixels),
                                       _ptr(gb), _ptr(gv), _ptr(gc), B, H, W, C, V, F, groups_ptr, ng,
                                       _ptr(dilated) if return_dilation else None)
    if rc != 0:
        raise RuntimeError('dirt_oracle_backward failed: %d' % rc)
    if not return_dilation:
        return gb, gv, gc
    return gb, gv, gc, list(dilated) if return_dilation == 'codes' else list((dilated & 3) >= 2)


class TriExport(ctypes.Structure):
    _fields_ = [('A', ctypes.c_int32 * 3), ('B', ctypes.c_int32 * 3), ('q', ctypes.c_int64 * 3),
                ('z', ctypes.c_float * 3), ('q0', ctypes.c_float * 3), ('q1', ctypes.c_float * 3),
                ('s', ctypes.c_float * 3), ('cref', ctypes.c_int32), ('rref', ctypes.c_int32),
                ('kind', ctypes.c_int32), ('bbox', ctypes.c_int32 * 4)]


def setup_records(vertices, faces, height, width):
    """Per-face setup records of ONE image (vertices [V,4], faces [F,3]) as a list of dicts."""
    vertices, faces = _f32(vertices), _i32(faces)
    V, F = vertices.shape[0], faces.shape[0]
    out = (TriExport * F)()
    lib().dirt_oracle_setup(_ptr(vertices), _ptr(faces), out, height, width, V, F)
    recs = []
    for e in out:
        recs.append(dict(kind=e.kind, A=list(e.A), B=list(e.B), q=list(e.q), z=list(e.z), q0=list(e.q0),
                         q1=list(e.q1), s=list(e.s), cref=e.cref, rref=e.rref, bbox=list(e.bbox)))
    return recs
