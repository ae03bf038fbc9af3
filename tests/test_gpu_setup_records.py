"""GPU: the triangle-setup kernel's output read straight out of the workspace and held to its contract by
tests/setup_records.py: every record field bit for bit against the oracle (the shading record's float64 sums to one fp32
rounding), every tile's references as an exact set, tile_count, the row lists, the large list, tile_flags and the
header.  A failure names the image, face or tile and the field.

Call modes: forward calls with C = 1, 3, 4 and 5 (C <= 4 writes the shading records, C = 3 carves the padded
colour-gradient rows); backward calls without the forward's workspace, which run setup for the records only (their
records must be the forward's, bit for bit), in the atomic and the deterministic backward pass; a workspace reused from
an earlier call on other geometry of the same sizes; a batch past the grid's 65535 images; the benched workload."""
import ctypes

import numpy as np
import pytest

import kernel_paths as kp
import setup_records as sr
from conftest import rel_close
from dirt_b200 import scenes
from test_gpu_paths import _p, _stream, abi_backward, abi_forward, abi_workspace

pytestmark = pytest.mark.gpu

CHANNELS = [1, 3, 4, 5]


# ---- scenes ---------------------------------------------------------------------------------------------------------------

def _square_with(faces=None, vertices=None):
    s = scenes.square_scene(32, 32, 16, 16, 8)
    if vertices is not None:
        s['vertices'] = np.concatenate([s['vertices'], vertices], axis=1)
        s['vertex_colors'] = np.concatenate([s['vertex_colors'], np.ones((1, vertices.shape[1], 1), np.float32)], axis=1)
    s['faces'] = faces if faces is not None else s['faces']
    return s


def _guard_band_soup():
    s = scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10, behind_camera=True)
    s['vertices'][:, ::7, 0] *= 4000.0   # far outside the guard band: hard faces in front of the eye
    return s


def _large_and_dense():
    """test_gpu_parity.test_large_faces_and_many_faces_per_tile: faces past SMALL_TILE_LIMIT tiles and 200 tiny ones."""
    rng = np.random.default_rng(4)
    s = scenes.random_soup(batch=1, width=96, height=80, n_faces=30, channels=3, seed=7)
    n = 200
    tiny = np.concatenate([rng.uniform(-0.12, 0.12, size=(n * 3, 2)), rng.uniform(-0.9, 0.9, size=(n * 3, 1)),
                           np.ones((n * 3, 1))], axis=1).astype(np.float32)
    V0 = s['vertices'].shape[1]
    s['vertices'] = np.concatenate([s['vertices'], tiny[None]], axis=1)
    s['vertex_colors'] = np.concatenate([s['vertex_colors'], rng.uniform(size=(1, n * 3, 3)).astype(np.float32)], axis=1)
    s['faces'] = np.concatenate([s['faces'], (V0 + np.arange(n * 3, dtype=np.int32)).reshape(1, n, 3)], axis=1)
    return s


SCENES = {
    'square': lambda: scenes.square_scene(width=64, height=48, centre_x=20, centre_y=30, size=12),
    'cylinder_batch2': lambda: scenes.cylinder_scene(batch=2, seed=3),
    'bent_square': lambda: scenes.bent_square_scene(channels=3),
    'cube': lambda: scenes.cube_scene(width=160, height=120),
    'soup_behind_camera': lambda: scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10,
                                                     behind_camera=True),
    'soup_guard_band': _guard_band_soup,
    'bad_faces': lambda: _square_with(np.concatenate([scenes.square_scene(32, 32, 16, 16, 8)['faces'],
                                                      np.array([[[0, 0, 1], [0, 1, 99], [-1, 1, 2]]], np.int32)], axis=1)),
    'nan_vertex': lambda: _square_with(np.array([[[0, 1, 2], [0, 2, 3], [0, 1, 4]]], np.int32),
                                       np.full((1, 1, 4), np.nan, np.float32)),
    'soup_13x7': lambda: scenes.random_soup(batch=1, width=13, height=7, n_faces=12, channels=3, seed=1),
    'soup_17x9': lambda: scenes.random_soup(batch=2, width=17, height=9, n_faces=20, channels=3, seed=5, behind_camera=True),
    'soup_1x1': lambda: scenes.random_soup(batch=1, width=1, height=1, n_faces=5, channels=1, seed=2),
    'large_and_dense': _large_and_dense,
    'bin_overflow': lambda: kp.bin_overflow_scene(batch=2),
    'coplanar_tie': lambda: kp.coplanar_tie_scene(batch=2),
    'edge_strip_8x65536': lambda: kp.edge_strip(8, 65536, 3, seed=1),
    'edge_strip_8x65537': lambda: kp.edge_strip(8, 65537, 3, seed=2),
    'edge_strip_65536x8': lambda: kp.edge_strip(65536, 8, 3, seed=3),
    'edge_strip_65537x8': lambda: kp.edge_strip(65537, 8, 3, seed=4),
    'cfg3_level1_batch3': lambda: scenes.config3(batch=3, width=96, height=80, level=1),
    'cfg3_level2_batch5': lambda: scenes.config3(batch=5, width=96, height=80, level=2),
    'no_faces': lambda: _square_with(np.zeros((1, 0, 3), np.int32)),
}


def with_channels(s, C, seed=0):
    """Scene `s` with a background and vertex colours of C channels (setup reads the colours only for its shading
    records)."""
    rng = np.random.default_rng(seed)
    B, H, W = s['background'].shape[:3]
    V = s['vertices'].shape[1]
    return dict(background=rng.uniform(size=(B, H, W, C)).astype(np.float32), vertices=s['vertices'],
                vertex_colors=rng.uniform(-1.0, 1.0, size=(B, V, C)).astype(np.float32), faces=s['faces'])


# ---- calls --------------------------------------------------------------------------------------------------------------

def _cuda(s):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.items()}


def _sizes(t):
    B, H, W, C = t['background'].shape
    return B, H, W, C, t['vertices'].shape[1], t['faces'].shape[1]


def _tag(t):
    B, H, W, C, V, F = _sizes(t)
    return sr.workspace_tag(t['vertices'].data_ptr(), t['faces'].data_ptr(), B, H, W, V, F)


def forward(L, t, workspace=None):
    """dirt_rasterise_forward -> (pixels, face ids, workspace), CUDA tensors."""
    import torch
    B, H, W = t['background'].shape[:3]
    pixels = torch.empty_like(t['background'])
    ids = torch.empty((B, H, W), dtype=torch.int32, device='cuda')
    ws = abi_forward(L, t['background'], t['vertices'], t['vertex_colors'], t['faces'], pixels, ids, workspace)
    return pixels, ids, ws


def visibility(L, t, workspace):
    import torch
    B, H, W, C, V, F = _sizes(t)
    ids = torch.empty((B, H, W), dtype=torch.int32, device='cuda')
    gbuffer = torch.empty((B, H, W, 4), dtype=torch.float32, device='cuda')
    rc = L.dirt_rasterise_visibility(_p(t['vertices']), _p(t['faces']), _p(ids), _p(gbuffer), B, H, W, V, F, _p(workspace),
                                     workspace.numel(), _stream())
    assert rc == 0, L.dirt_error_string(rc)
    return ids, gbuffer


def backward(L, t, pixels, grad_pixels, ids, workspace=None, holds_setup=False, deterministic=False):
    """dirt_rasterise_backward_ex or dirt_rasterise_backward_deterministic with the given face ids ->
    (grad_background, grad_vertices, grad_vertex_colors, the workspace)."""
    import torch
    B, H, W, C, V, F = _sizes(t)
    ws = abi_workspace(L, B, H, W, C, V, F) if workspace is None else workspace
    gb, gv, gc = torch.empty_like(pixels), torch.empty((B, V, 4), device='cuda'), torch.empty((B, V, C), device='cuda')
    if not deterministic:
        abi_backward(L, t['vertices'], t['faces'], pixels, grad_pixels, ids, gb, gv, gc, workspace=ws, holds_setup=holds_setup)
        return gb, gv, gc, ws
    n = max(int(L.dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F)), 256)
    scratch = torch.empty(n, dtype=torch.uint8, device='cuda')
    rc = L.dirt_rasterise_backward_deterministic(_p(t['vertices']), _p(t['faces']), _p(pixels), _p(grad_pixels), _p(ids),
                                                 _p(gb), _p(gv), _p(gc), B, H, W, C, V, F, None, 0, int(holds_setup), 0,
                                                 _p(ws), ws.numel(), _p(scratch), n, _stream())
    assert rc == 0, L.dirt_error_string(rc)
    return gb, gv, gc, ws


def _np(x):
    return x.cpu().numpy()


def check_forward(t, s, ids, ws, stats=None, images=None):
    B, H, W, C, V, F = _sizes(t)
    msg = sr.check(_np(ws), s['vertices'], s['faces'], H, W, C, vertex_colors=s['vertex_colors'], face_ids=_np(ids),
                   tag=_tag(t), images=images, stats=stats)
    assert msg is None, msg


# ---- tests ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('C', CHANNELS)
@pytest.mark.parametrize('name', list(SCENES))
def test_forward_setup_output(cuda_lib, oracle, name, C):
    s = with_channels(SCENES[name](), C, seed=C)
    t = _cuda(s)
    _, ids, ws = forward(cuda_lib, t)
    stats = {}
    check_forward(t, s, ids, ws, stats)
    if name == 'bin_overflow':
        # the spill path: a bin past BIN_CAP, a row list past OVF_ROW_CAP, small faces in the large list
        assert stats['bins_past_cap'] > 0 and stats['rows_past_cap'] > 0 and stats['faces_spilled_to_large'] > 0, stats
    if C <= 4 and 'shade_ratio' in stats:
        print('%s C=%d: worst TriShade error %.3f of one fp32 rounding' % (name, C, stats['shade_ratio']))


@pytest.mark.parametrize('deterministic', [False, True], ids=['atomic', 'deterministic'])
@pytest.mark.parametrize('name', list(SCENES))
def test_backward_records_only(cuda_lib, oracle, name, deterministic):
    """A backward call handed face ids but not the forward's workspace runs setup for the records only: TriCov,
    TriInterp and TriXY as the forward's, bit for bit, and a header naming its own geometry."""
    import torch
    s = with_channels(SCENES[name](), 3)
    t = _cuda(s)
    pixels, ids, ws_f = forward(cuda_lib, t)
    gp = torch.from_numpy(np.random.default_rng(0).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
    *_, ws_b = backward(cuda_lib, t, pixels, gp, ids, deterministic=deterministic)
    B, H, W, C, V, F = _sizes(t)
    msg = sr.check(_np(ws_b), s['vertices'], s['faces'], H, W, C, lists=False, shade=False, tag=_tag(t))
    assert msg is None, msg
    fwd, bwd = sr.read_workspace(_np(ws_f), B, H, W, C, V, F), sr.read_workspace(_np(ws_b), B, H, W, C, V, F)
    for block in ('cov_large', 'itp', 'xy'):
        np.testing.assert_array_equal(bwd[block].view(np.uint8), fwd[block].view(np.uint8), err_msg=block)


def _shifted(s, dx):
    """Scene `s` moved by dx in NDC, its faces in reverse order: other geometry of the same sizes."""
    out = dict(s)
    v = s['vertices'].copy()
    v[..., 0] += np.float32(dx) * v[..., 3]
    out['vertices'] = v
    out['faces'] = np.ascontiguousarray(s['faces'][:, ::-1])
    return out


REUSED = {
    'bin_overflow': (lambda: kp.bin_overflow_scene(batch=2), lambda: _shifted(kp.bin_overflow_scene(batch=2), 0.21)),
    'bin_overflow_after_light': (lambda: _shifted(kp.bin_overflow_scene(batch=2, n=1200, second=1200), -0.3),
                                 lambda: kp.bin_overflow_scene(batch=2)),
    'cfg3_level2_batch5': (lambda: scenes.config3(batch=5, width=96, height=80, level=2, seed=1),
                           lambda: scenes.config3(batch=5, width=96, height=80, level=2, seed=2)),
    'soup_behind_camera': (lambda: scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10,
                                                      behind_camera=True),
                           lambda: scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=11,
                                                      behind_camera=True)),
    'coplanar_tie': (lambda: kp.coplanar_tie_scene(batch=2, seed=0), lambda: kp.coplanar_tie_scene(batch=2, seed=1)),
}


@pytest.mark.parametrize('C', [3, 4])
@pytest.mark.parametrize('name', list(REUSED))
def test_reused_workspace(cuda_lib, oracle, name, C):
    """Scene B on the workspace a call on scene A (same sizes, other geometry) left behind: B's setup output passes the
    checker, and its face ids, pixels, G-buffer and gradients are those of a call on a fresh workspace, bit for bit (the
    atomic backward pass's vertex gradients, whose summation order varies, to rel_close)."""
    import torch
    sa, sb = (with_channels(f(), C, seed=C) for f in REUSED[name])
    ta, tb = _cuda(sa), _cuda(sb)
    gp = torch.from_numpy(np.random.default_rng(1).standard_normal(sb['background'].shape).astype(np.float32)).cuda()

    # fresh workspaces
    px_f, ids_f, ws_f = forward(cuda_lib, tb)
    vis_ids_f, gbuf_f = visibility(cuda_lib, tb, abi_workspace(cuda_lib, *_sizes(tb)))
    det_f = backward(cuda_lib, tb, px_f, gp, ids_f, ws_f, holds_setup=True, deterministic=True)
    atom_f = backward(cuda_lib, tb, px_f, gp, ids_f, ws_f, holds_setup=True)

    # scene A's forward call first, then B on its workspace
    ws = forward(cuda_lib, ta)[2]
    px, ids, _ = forward(cuda_lib, tb, ws)
    check_forward(tb, sb, ids, ws)
    det = backward(cuda_lib, tb, px, gp, ids, ws, holds_setup=True, deterministic=True)
    atom = backward(cuda_lib, tb, px, gp, ids, ws, holds_setup=True)
    ws_v = abi_workspace(cuda_lib, *_sizes(ta))
    visibility(cuda_lib, ta, ws_v)
    vis_ids, gbuf = visibility(cuda_lib, tb, ws_v)

    for what, a, b in (('face ids', ids, ids_f), ('pixels', px, px_f), ('visibility face ids', vis_ids, vis_ids_f),
                       ('G-buffer', gbuf, gbuf_f), ('grad_background', atom[0], atom_f[0]),
                       ('deterministic grad_background', det[0], det_f[0]), ('deterministic grad_vertices', det[1], det_f[1]),
                       ('deterministic grad_vertex_colors', det[2], det_f[2])):
        np.testing.assert_array_equal(_np(a).view(np.uint32), _np(b).view(np.uint32), err_msg='%s: %s' % (name, what))
    for what, a, b in (('grad_vertices', atom[1], atom_f[1]), ('grad_vertex_colors', atom[2], atom_f[2])):
        ok, ratio = rel_close(_np(a), _np(b))
        assert ok, '%s: %s off by %.2fx the tolerance' % (name, what, ratio)


def test_no_faces_through_autograd(cuda_lib):
    """A mesh without faces through rasterise_batch and autograd: the backward pass reuses the forward's workspace,
    whose header must carry the forward's tag even though there was no face to set up.  The vertex gradients are 0."""
    import torch
    import dirt_b200 as dirt
    s = with_channels(SCENES['no_faces'](), 3)
    t = _cuda(s)
    for k in ('background', 'vertices', 'vertex_colors'):
        t[k].requires_grad_(True)
    pixels = dirt.rasterise_batch(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    pixels.sum().backward()
    assert torch.equal(pixels.detach(), t['background'].detach())
    assert torch.equal(t['background'].grad, torch.ones_like(pixels))
    assert not t['vertices'].grad.any() and not t['vertex_colors'].grad.any()


def test_batch_past_the_grid_limit(cuda_lib, oracle):
    """65544 images of two faces (test_gpu_paths.test_batch_past_the_grid_limit): the records and lists of the first
    and the last images, past gridDim's 65535."""
    s = kp.grid_limit_scene()
    t = _cuda(s)
    _, ids, ws = forward(cuda_lib, t)
    B = s['background'].shape[0]
    images = list(range(4)) + list(range(65530, B))
    check_forward(t, s, ids, ws, images=images)


def test_benched_workload(cuda_lib, oracle):
    """cfg3 as bench.py runs it: 64 images of 512 x 512, C = 4, icosphere-4 (5120 faces each)."""
    s = scenes.config3()
    t = _cuda(s)
    _, ids, ws = forward(cuda_lib, t)
    stats = {}
    check_forward(t, s, ids, ws, stats)
    print('cfg3: %s' % stats)
