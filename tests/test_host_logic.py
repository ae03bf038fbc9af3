"""CPU: host-side logic of the drop-in boundary (no kernel is launched)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_channel_groups_follow_the_reference():
    from dirt_b200.rasterise_ops import default_channel_groups
    # dirt/rasterise_ops.py:80-108: 1 or 3 -> single op; else groups of 3 while >= 3 remain, then 1s
    assert default_channel_groups(1) == [1]
    assert default_channel_groups(3) == [3]
    assert default_channel_groups(2) == [1, 1]
    assert default_channel_groups(4) == [3, 1]
    assert default_channel_groups(5) == [3, 1, 1]
    assert default_channel_groups(7) == [3, 3, 1]
    assert default_channel_groups(10) == [3, 3, 3, 1]
    with pytest.raises(ValueError):
        default_channel_groups(0)


def test_library_exports_every_declared_symbol():
    from dirt_b200 import build, _lib
    build.build()
    header = open(os.path.join(ROOT, 'include', 'dirt_b200.h')).read()
    declared = set(re.findall(r'\b(dirt_[a-z_]+)\s*\(', header))
    assert declared == set(_lib.EXPORTED_SYMBOLS)
    lib = ctypes.CDLL(build.SO_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    L = _lib.lib()
    assert L.dirt_abi_version() == 4
    assert _lib.error_string(0) == 'ok'
    assert 'workspace' in _lib.error_string(-3)
    # workspace size is a pure function of the sizes and grows with them
    a = L.dirt_workspace_bytes(1, 64, 64, 3, 100, 200)
    b = L.dirt_workspace_bytes(2, 64, 64, 3, 100, 200)
    assert 0 < a < b
    assert L.dirt_workspace_bytes(1, 0, 64, 3, 100, 200) == 0
    # the smaller size leaves out exactly the face-id scratch block (B*H*W int32, 256-byte granules)
    assert a - L.dirt_workspace_bytes_min(1, 64, 64, 3, 100, 200) == 64 * 64 * 4
    assert L.dirt_workspace_bytes_min(1, 0, 64, 3, 100, 200) == 0


def test_argument_validation_without_a_gpu():
    # shape errors are reported before anything touches the device, with the reference's wording
    import dirt_b200 as dirt
    bg = torch.zeros(2, 8, 8, 3)
    verts = torch.zeros(2, 5, 4)
    cols = torch.zeros(2, 5, 3)
    faces = torch.zeros(2, 4, 3, dtype=torch.int32)
    with pytest.raises(ValueError, match='vertices to be 3D'):
        dirt.rasterise_batch(bg, torch.zeros(2, 5, 3), cols, faces)
    with pytest.raises(ValueError, match='vertex_colors to be 3D'):
        dirt.rasterise_batch(bg, verts, torch.zeros(2, 5, 4), faces)
    with pytest.raises(ValueError, match='faces to be 3D'):
        dirt.rasterise_batch(bg, verts, cols, torch.zeros(2, 4, 4, dtype=torch.int32))
    with pytest.raises(ValueError, match='same leading'):
        dirt.rasterise_batch(bg, verts[:1], cols, faces)
    with pytest.raises(ValueError, match='background_tensor to be 4D'):
        dirt.rasterise_batch(bg, verts, cols, faces, height=16)
    if not torch.cuda.is_available():
        # no CPU kernel exists (csrc/rasterise_egl.cpp:410); the product never falls back to one
        with pytest.raises(RuntimeError, match='CUDA'):
            dirt.rasterise_batch(bg, verts, cols, faces)


def test_c_abi_rejects_bad_arguments():
    from dirt_b200 import _lib
    L = _lib.lib()
    null = ctypes.c_void_p(0)
    assert L.dirt_rasterise_forward(null, null, null, null, null, null, 1, 0, 8, 3, 4, 2, null, 0, null) == _lib.ERR_BAD_SHAPE
    assert L.dirt_rasterise_forward(null, null, null, null, null, null, 1, 8, 8, 3, 4, 2, null, 0, null) == _lib.ERR_NULL_POINTER
    groups = (ctypes.c_int * 2)(2, 2)
    assert L.dirt_rasterise_backward(null, null, null, null, null, null, null, null, 1, 8, 8, 4, 4, 2, groups, 2, 0, null, 0,
                                     null) == _lib.ERR_BAD_CHANNEL_GROUPS
    assert L.dirt_rasterise_backward(null, null, null, null, null, null, null, null, 1, 8, 8, 3, (1 << 24) + 1, 2, None, 0,
                                     0, null, 0, null) == _lib.ERR_TOO_MANY_VERTICES
    # a backward call without face ids needs the full workspace, one with face ids the smaller one (checked before any
    # pointer is touched: the addresses below are never dereferenced)
    p = lambda a: ctypes.c_void_p(a)
    small, full = L.dirt_workspace_bytes_min(1, 8, 8, 3, 4, 2), L.dirt_workspace_bytes(1, 8, 8, 3, 4, 2)
    assert small < full
    args = lambda ids, nbytes: (p(4096), p(4096), p(4096), p(4096), ids, p(4096), p(4096), p(4096), 1, 8, 8, 3, 4, 2, None, 0, 0,
                                p(4096), nbytes, null)
    assert L.dirt_rasterise_backward(*args(null, small)) == _lib.ERR_WORKSPACE_TOO_SMALL
    assert L.dirt_rasterise_backward(*args(p(4096), small - 1)) == _lib.ERR_WORKSPACE_TOO_SMALL
    # the peer exchange validates its arguments before it launches anything
    assert L.dirt_peer_exchange_bytes(8, 20496) == 2 * 8 * 20496 * 4 and L.dirt_peer_exchange_bytes(17, 4) == 0
    two = (ctypes.c_void_p * 2)(p(4096), p(4096))
    assert L.dirt_peer_exchange(p(4096), p(8192), two, two, 2, 0, 6, 1, null) == _lib.ERR_BAD_SHAPE      # count % 4
    assert L.dirt_peer_exchange(p(4096), p(4096), two, two, 2, 0, 8, 1, null) == _lib.ERR_BAD_SHAPE      # local == out
    assert L.dirt_peer_exchange(p(4096), p(8192), two, two, 2, 2, 8, 1, null) == _lib.ERR_BAD_SHAPE      # rank >= world
    assert L.dirt_peer_exchange(p(4096), p(8192), two, two, 2, 0, 8, 0, null) == _lib.ERR_BAD_SHAPE      # sequence 0
    assert L.dirt_peer_exchange(p(4100), p(8192), two, two, 2, 0, 8, 1, null) == _lib.ERR_MISALIGNED
    assert L.dirt_peer_exchange(null, p(8192), two, two, 2, 0, 8, 1, null) == _lib.ERR_NULL_POINTER
    # B == 0 is a no-op, as an empty batch is for the reference
    assert L.dirt_rasterise_forward(null, null, null, null, null, null, 0, 8, 8, 3, 4, 2, null, 0, null) == 0
    # channel counts whose greedy split into groups of 3 and 1 would not fit the group table are a shape error up front
    # (384 = 128 groups of 3 fits, 383 = 127 + 2 does not), the same answer from forward and backward
    assert L.dirt_workspace_bytes(1, 8, 8, 384, 4, 2) > 0 and L.dirt_workspace_bytes(1, 8, 8, 383, 4, 2) == 0
    assert L.dirt_rasterise_backward(null, null, null, null, null, null, null, null, 1, 8, 8, 383, 4, 2, None, 0, 0, null, 0,
                                     null) == _lib.ERR_BAD_SHAPE
    # unknown flag bits of the extended backward entry point
    assert L.dirt_rasterise_backward_ex(null, null, null, null, null, null, null, null, 1, 8, 8, 3, 4, 2, None, 0, 0, 64,
                                        null, 0, null) == _lib.ERR_BAD_SHAPE


def test_matrices_and_lighting_helpers():
    from dirt_b200 import matrices, lighting, scenes
    np.testing.assert_allclose(matrices.rodrigues([0., 0.5, 0.]).numpy(), scenes.rodrigues([0., 0.5, 0.]), atol=1e-6)
    np.testing.assert_allclose(matrices.perspective_projection(0.1, 20., 0.1, 0.75).numpy(),
                               scenes.perspective_projection(0.1, 20., 0.1, 0.75), atol=1e-6)
    np.testing.assert_allclose(matrices.compose(matrices.translation([0., -1.5, -3.5]), matrices.rodrigues([-0.3, 0., 0.])).numpy(),
                               scenes.translation([0., -1.5, -3.5]) @ scenes.rodrigues([-0.3, 0., 0.]), atol=1e-6)
    v, f = scenes.icosphere(1)
    n = lighting.vertex_normals(torch.from_numpy(v), torch.from_numpy(f)).numpy()
    np.testing.assert_allclose(n, v / np.linalg.norm(v, axis=1, keepdims=True), atol=5e-2)   # sphere normals ~ positions
    sv, sf = lighting.split_vertices_by_face(torch.from_numpy(v), torch.from_numpy(f))
    assert sv.shape == (f.shape[0] * 3, 3) and sf.shape == f.shape
    flat = lighting.vertex_normals_pre_split(sv, sf)
    assert torch.allclose(flat[0], flat[1]) and torch.allclose(flat[1], flat[2])
    lit = lighting.diffuse_directional(torch.from_numpy(n), torch.ones(v.shape[0], 3), [1., 0., 0.], [1., 1., 1.])
    assert lit.shape == (v.shape[0], 3) and float(lit.min()) >= 0.


def test_bench_reference_arm_prints_one_json_line():
    """bench.py --impl reference runs the CPU port (no GPU needed) and must put exactly one JSON line on stdout,
    with the keys the contract names."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    proc = subprocess.run([sys.executable, os.path.join(root, 'bench.py'), '--impl', 'reference', '--workload', 'cfg2',
                           '--steps', '1', '--warmup', '0', '--cpu-sample', '1'],
                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300, check=True)
    lines = [ln for ln in proc.stdout.decode().splitlines() if ln.strip()]
    assert len(lines) == 1, lines
    out = json.loads(lines[0])
    assert out['impl'] == 'reference' and out['metric'] == 'fwd+bwd Mpixels/sec' and out['unit'] == 'Mpixels/s'
    for key in ('value', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling', 'dtype', 'data', 'config',
                'cpu_baseline', 'e2e'):
        assert key in out, key
    assert out['value'] > 0 and out['cpu_baseline']['kind'] == 'port' and out['e2e']['h2d_bytes_per_step'] == 0


def test_reference_gradient_library_is_built():
    """Where a reference checkout can be found, __graft_entry__.build() compiles the reference's gradient kernel into
    oracle/_ref/libdirt_ref_grad.so, which tests/test_gpu_ref_live.py runs against the CUDA path; a build() that quietly
    stopped producing it would turn those tests into skips."""
    from oracle import ref
    if not ref.can_build():
        pytest.skip('no reference checkout (neither $DIRT_REFERENCE nor a `reference` directory beside the repository)')
    so = os.path.join(ROOT, 'oracle', '_ref', 'libdirt_ref_grad.so')
    assert os.path.exists(so), '%s is missing although a reference checkout is at %s' % (so, ref.reference_checkout())
    lib = ctypes.CDLL(so)
    for name in ('dirt_ref_assemble_grads', 'dirt_ref_upload_vertices', 'dirt_ref_sizeof_vertex'):
        assert hasattr(lib, name), name


def test_reference_inputs_and_oracle_dilation_masks():
    """The host side of the live reference comparison: the vertex-index image the reference's fragment shader would
    write, and the oracle's dilation masks (one per channel group, the same gradients as without them)."""
    from dirt_b200 import scenes
    from oracle import oracle, ref
    s = scenes.random_soup(batch=3, width=33, height=27, n_faces=40, channels=4, seed=4)
    ids, _ = oracle.visibility(s['vertices'], s['faces'], 27, 33)
    vids = ref.vertex_ids_image(s['faces'], ids)
    for b in range(3):
        for r, c in zip(*np.nonzero(ids[b] >= 0)):
            assert (vids[b, r, c] == s['faces'][b, ids[b, r, c]]).all()
        assert (vids[b][ids[b] < 0] == -1).all()
    pixels = oracle.forward(**s)
    gp = np.random.default_rng(2).standard_normal(pixels.shape).astype(np.float32)
    plain = oracle.backward(s['vertices'], s['faces'], pixels, gp, [1, 3])
    gb, gv, gc, masks = oracle.backward(s['vertices'], s['faces'], pixels, gp, [1, 3], return_dilation=True)
    for a, b in zip(plain, (gb, gv, gc)):
        np.testing.assert_array_equal(a, b)
    assert len(masks) == 2 and all(m.shape == ids.shape and m.dtype == bool for m in masks)
    for m in masks:
        assert m.any()
        # dilation happens at interior pixels only (csrc/rasterise_grad_egl.cu:155)
        assert not (m[:, 0].any() or m[:, -1].any() or m[:, :, 0].any() or m[:, :, -1].any())
    assert len(oracle.backward(s['vertices'], s['faces'], pixels, gp, return_dilation=True)[3]) == 2   # greedy [3, 1]
