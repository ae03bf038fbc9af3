"""ctypes wrapper around oracle/_ref/libdirt_ref_grad.so: the REFERENCE'S OWN gradient kernel.

TEST INFRASTRUCTURE ONLY.  oracle/Makefile (target `ref`) compiles the reference's csrc/rasterise_grad_egl.cu
UNMODIFIED, against the stand-in TensorFlow headers in oracle/ref_shim/, into oracle/_ref/ (git-ignored).  It needs
a GPU to run: `assemble_grads` is CUDA.  What it pins: every gradient
value and every dilation decision of csrc/rasterise_grad_egl.cu:93-236, given a G-buffer.  The G-buffer itself (what
the OpenGL driver renders in the reference) is an input -- the CPU oracle's.

Two users: tests/golden/make_ref_golden.py stores the kernel's outputs under tests/golden/ (what CPU-only boxes compare
with), and tests/test_gpu_ref_live.py runs the library live on the GPU against the CUDA path.  __graft_entry__.build()
builds the library whenever a reference checkout can be found: $DIRT_REFERENCE, or else a directory named `reference`
beside the repository root.  The GPU tests only load what build() left; they never read the checkout.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, '_ref', 'libdirt_ref_grad.so')
_lib = None

BAD_ARGS = -1000           # ref_driver.cu DIRT_REF_BAD_ARGS
FRAME_TOO_LARGE = -1001    # ref_driver.cu DIRT_REF_FRAME_TOO_LARGE


class FrameTooLarge(RuntimeError):
    """The tiled framebuffer of a call is larger than the device's 2D surface limits; nothing ran."""


def reference_checkout():
    """The reference checkout (of pmh47/dirt) to build from: $DIRT_REFERENCE if set, else a directory named
    `reference` beside the repository root.  None if that directory does not hold csrc/rasterise_grad_egl.cu."""
    path = os.environ.get('DIRT_REFERENCE', '') or os.path.join(os.path.dirname(os.path.dirname(_HERE)), 'reference')
    return path if os.path.exists(os.path.join(path, 'csrc', 'rasterise_grad_egl.cu')) else None


def can_build():
    return reference_checkout() is not None


def build(force=False):
    """make -C oracle ref with the checkout of reference_checkout(); raises if there is none or nvcc fails."""
    checkout = reference_checkout()
    if checkout is None:
        raise RuntimeError('no reference checkout: set DIRT_REFERENCE to a checkout of pmh47/dirt to build oracle/_ref')
    if force and os.path.exists(_SO):
        os.remove(_SO)
    proc = subprocess.run(['make', '-C', _HERE, 'ref', 'REFERENCE=' + os.path.abspath(checkout)], capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError('building oracle/_ref failed:\n' + proc.stdout + proc.stderr)
    return _SO


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError('%s is missing (build it with __graft_entry__.build() or '
                               '`make -C oracle ref REFERENCE=<checkout of pmh47/dirt>`)' % _SO)
        _lib = ctypes.CDLL(_SO)
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def vertex_ids_image(faces, face_ids):
    """[B,H,W,3] int32: the three vertex indices of each pixel's visible face, -1 where uncovered
    (what the reference's backward fragment shader writes, csrc/shaders.cpp:62-76)."""
    faces = np.asarray(faces, np.int32)
    face_ids = np.asarray(face_ids, np.int32)
    B = face_ids.shape[0]
    covered = face_ids >= 0
    if faces.shape[1] == 0:
        return np.full(face_ids.shape + (3,), -1, np.int32)
    idx = np.where(covered, face_ids, 0).reshape(B, -1, 1)
    out = np.take_along_axis(faces, np.repeat(idx, 3, axis=2), axis=1).reshape(face_ids.shape + (3,))
    return np.where(covered[..., None], out, np.int32(-1)).astype(np.int32)


def assemble_grads(gbuffer, vertex_ids, pixels, grad_pixels, vertices, with_debug=False, split=1):
    """ONE native RasteriseGrad call (C = 1 or 3) of the reference kernel.
    -> grad_background [B,H,W,C], grad_vertices [B,V,4], grad_vertex_colors [B,V,C] (, debug_thingy [B,H,W,3]).
    With split > 1: split^2 runs of the kernel, each with grad_pixels kept on one (row % split, col % split) lattice of
    pixels, their vertex gradients summed in float64 (ref_driver.cu assemble).  The per-pixel terms are the kernel's
    own; only its order-dependent fp32 atomic sums are made split^2 times shorter."""
    gbuffer, pixels, grad_pixels, vertices = _f32(gbuffer), _f32(pixels), _f32(grad_pixels), _f32(vertices)
    vertex_ids = np.ascontiguousarray(vertex_ids, np.int32)
    B, H, W, C = pixels.shape
    V = vertices.shape[1]
    assert C in (1, 3) and gbuffer.shape == (B, H, W, 4) and vertex_ids.shape == (B, H, W, 3)
    assert grad_pixels.shape == pixels.shape and vertices.shape == (B, V, 4)
    acc = np.float64 if split > 1 else np.float32
    gv = np.empty((B, V, 4), acc)
    gc = np.empty((B, V, C), acc)
    gb = np.empty((B, H, W, C), np.float32)
    dbg = np.empty((B, H, W, 3), np.float32) if with_debug else None
    args = (_ptr(gbuffer), _ptr(vertex_ids), _ptr(pixels), _ptr(grad_pixels), _ptr(vertices), _ptr(gv), _ptr(gc), _ptr(gb),
            _ptr(dbg) if with_debug else None, B, H, W, C, V)
    if split > 1:
        rc = lib().dirt_ref_assemble_grads_split(*args, int(split))
    else:
        rc = lib().dirt_ref_assemble_grads(*args)
    if rc == FRAME_TOO_LARGE:
        raise FrameTooLarge('dirt_ref_assemble_grads: %d frames of %d x %d do not fit in one 2D surface' % (B, W, H))
    if rc != 0:
        raise RuntimeError('dirt_ref_assemble_grads failed: %d' % rc)
    return (gb, gv, gc, dbg) if with_debug else (gb, gv, gc)


# what assemble_grads writes into debug_thingy[..., 0] where a pixel took a neighbour's face (csrc/rasterise_grad_egl.cu:172)
DILATION_MARK = np.float32(1e-2)


def backward(vertices, faces, pixels, grad_pixels, gbuffer, face_ids, channel_groups=None, return_dilation=False, split=1):
    """The Python-level gradient of the reference for any channel count: one native call per channel group on a
    contiguous slice, grad_vertices summed over groups, the others concatenated
    (dirt/rasterise_ops.py:86-108,111-129; the explicit form is _rasterise_grad_multichannel, :132-177).
    With return_dilation, also a list with one bool [B,H,W] mask per channel group: the pixels where the kernel took
    a neighbour's face (debug_thingy[..., 0] == 1e-2; the launcher clears it to 0 before the kernel runs).
    `split` > 1: see assemble_grads; grad_vertices and grad_vertex_colors then come back as float64."""
    from . import oracle
    pixels, grad_pixels = _f32(pixels), _f32(grad_pixels)
    C = pixels.shape[-1]
    groups = list(channel_groups) if channel_groups is not None else oracle.default_groups(C)
    assert sum(groups) == C
    vids = vertex_ids_image(faces, face_ids)
    gbs, gcs, masks, gv_total, begin = [], [], [], None, 0
    for width in groups:
        sl = slice(begin, begin + width)
        out = assemble_grads(gbuffer, vids, np.ascontiguousarray(pixels[..., sl]),
                             np.ascontiguousarray(grad_pixels[..., sl]), vertices, with_debug=return_dilation, split=split)
        gb, gv, gc = out[:3]
        if return_dilation:
            masks.append(out[3][..., 0] == DILATION_MARK)
        gbs.append(gb)
        gcs.append(gc)
        gv_total = gv if gv_total is None else gv_total + gv
        begin += width
    result = (np.concatenate(gbs, axis=-1), gv_total, np.concatenate(gcs, axis=-1))
    return result + (masks,) if return_dilation else result


def upload_vertices(vertices, faces):
    """The reference's vertex expansion kernel (csrc/rasterise_grad_egl.cu:12-34): structured array [B, 3F]."""
    vertices = _f32(vertices)
    faces = np.ascontiguousarray(faces, np.int32)
    B, V, _ = vertices.shape
    F = faces.shape[1]
    dt = np.dtype([('position', np.float32, 4), ('barycentric', np.float32, 2), ('indices', np.int32, 3)])
    assert dt.itemsize == lib().dirt_ref_sizeof_vertex()
    out = np.empty((B, 3 * F), dt)
    rc = lib().dirt_ref_upload_vertices(_ptr(vertices), _ptr(faces), _ptr(out), B, V, F)
    if rc != 0:
        raise RuntimeError('dirt_ref_upload_vertices failed: %d' % rc)
    return out
