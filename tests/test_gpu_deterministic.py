"""GPU: the deterministic backward pass (dirt_rasterise_backward_deterministic) against the CPU oracle at the bars of
test_gpu_parity.py, its dilation codes against the oracle's dilation masks, its reproducibility (two calls, CUDA graph
replay, an item alone against the same item in a batch) and its routing through the public API under
torch.use_deterministic_algorithms."""
import ctypes

import numpy as np
import pytest

import kernel_paths as kp
from conftest import rel_close
from dirt_b200 import scenes

pytestmark = pytest.mark.gpu

FLAGS = list(range(8))   # every combination of DIRT_BWD_SHARED_GEOMETRY = 1, _SKIP_POSITION = 2, _SKIP_COLOUR = 4


def _cuda(s):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.items()}


def _groups_arg(groups):
    if groups is None:
        return None, 0
    return (ctypes.c_int * len(groups))(*groups), len(groups)


def det_call(t, pixels, gp, ids=None, groups=None, flags=0, ws=None, holds_setup=0, out=None, scratch=None):
    """One dirt_rasterise_backward_deterministic call on CUDA tensors -> (gb, gv, gc, scratch)."""
    import torch
    from dirt_b200 import _lib
    from dirt_b200 import rasterise_ops as ops
    L = _lib.lib()
    B, H, W, C = pixels.shape
    V, F = t['vertices'].shape[1], t['faces'].shape[1]
    lead = () if flags & 1 else (B,)
    if out is None:
        out = (torch.full_like(pixels, 7.0), torch.full(lead + (V, 4), 7.0, device='cuda'),
               torch.full(lead + (V, C), 7.0, device='cuda'))
    gb, gv, gc = out
    if ws is None:
        ws, _ = ops._workspace(B, H, W, C, V, F, pixels.device, face_id_scratch=ids is None)
    nbytes = int(L.dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F))
    if scratch is None:
        scratch = torch.empty(max(nbytes, 256), dtype=torch.uint8, device='cuda')
    g, n = _groups_arg(groups)
    rc = L.dirt_rasterise_backward_deterministic(
        ops._ptr(t['vertices']), ops._ptr(t['faces']), ops._ptr(pixels), ops._ptr(gp), ops._ptr(ids), ops._ptr(gb),
        ops._ptr(gv), ops._ptr(gc), B, H, W, C, V, F, g, n, holds_setup, flags, ops._ptr(ws), int(ws.numel()),
        ops._ptr(scratch), int(scratch.numel()), ops._stream_ptr(pixels.device))
    _lib.check(rc, 'RasteriseGrad')
    return gb, gv, gc, scratch


def codes(scratch, B, H, W, n_groups):
    px = B * H * W
    return scratch[:n_groups * px].view(n_groups, B, H, W).cpu().numpy()


def check_against_oracle(oracle, s, seed=0, groups=None, label='', ids_modes=('given', 'derived')):
    import torch
    from dirt_b200 import rasterise_ops as ops
    t = _cuda(s)
    pixels_o, ids_o = oracle.forward(**s, return_face_ids=True)
    gp = np.random.default_rng(seed).standard_normal(pixels_o.shape).astype(np.float32)
    gb_o, gv_o, gc_o, masks = oracle.backward(s['vertices'], s['faces'], pixels_o, gp, groups, return_dilation=True)
    pixels, gp_t = torch.from_numpy(pixels_o).cuda(), torch.from_numpy(gp).cuda()
    B, H, W, C = pixels_o.shape
    for mode in ids_modes:
        ids = torch.from_numpy(ids_o).cuda() if mode == 'given' else None
        gb, gv, gc, scratch = det_call(t, pixels, gp_t, ids, groups)
        np.testing.assert_array_equal(gb.cpu().numpy(), gb_o, err_msg=label + ': grad_background differs')
        for name, a, b in (('grad_vertices', gv, gv_o), ('grad_vertex_colors', gc, gc_o)):
            ok, ratio = rel_close(a.cpu().numpy(), b, name='deterministic ' + name + ' vs oracle')
            assert ok, '%s (%s ids): %s off by %.2fx the tolerance' % (label, mode, name, ratio)
        assert (gv[..., 2] == 0).all()
        n = len(masks)
        cp = codes(scratch, B, H, W, n)
        for g in range(n):
            np.testing.assert_array_equal((cp[g] & 3) >= 2, np.asarray(masks[g], bool), err_msg=label + ': dilation of group %d' % g)
    # the forward call's workspace handed over, as the autograd node does
    _, ids_g, ws = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'], return_workspace=True)
    gb, gv, gc, _ = det_call(t, pixels, gp_t, ids_g, groups, ws=ws, holds_setup=1)
    np.testing.assert_array_equal(gb.cpu().numpy(), gb_o)
    assert rel_close(gv.cpu().numpy(), gv_o)[0] and rel_close(gc.cpu().numpy(), gc_o)[0], label + ': workspace reuse'
    ops.workspace_status(ws, B, H, W, C, t['vertices'].shape[1], t['faces'].shape[1])


@pytest.mark.parametrize('name,kwargs', [
    ('square_scene', dict(width=64, height=48, centre_x=20, centre_y=30, size=12)),
    ('cylinder_scene', dict(batch=2, seed=3)),
    ('bent_square_scene', dict(channels=1)),
    ('bent_square_scene', dict(channels=4)),
    ('bent_square_scene', dict(channels=7)),
    ('bent_square_scene', dict(channels=2, width=37, height=29)),
    ('cube_scene', dict(width=160, height=120)),
    ('config2', dict()),
])
def test_reference_scenes(cuda_lib, oracle, name, kwargs):
    check_against_oracle(oracle, getattr(scenes, name)(**kwargs), label=name)


@pytest.mark.parametrize('seed', [0, 1])
@pytest.mark.parametrize('channels', [1, 3, 4, 5])
def test_random_soup(cuda_lib, oracle, seed, channels):
    s = scenes.random_soup(batch=2, width=61, height=45, n_faces=70, channels=channels, seed=seed)
    check_against_oracle(oracle, s, seed=seed, label='soup')


@pytest.mark.parametrize('seed', [0, 1])
def test_behind_camera_and_guard_band(cuda_lib, oracle, seed):
    s = scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10 + seed, behind_camera=True)
    check_against_oracle(oracle, s, seed=seed, label='behind-camera soup')
    s['vertices'][:, ::7, 0] *= 4000.0
    check_against_oracle(oracle, s, seed=seed, label='guard-band soup')


@pytest.mark.parametrize('channels,groups', [(1, None), (2, [1, 1]), (4, [1, 3]), (4, [1, 1, 1, 1]), (5, [3, 1, 1]),
                                             (5, [1, 3, 1]), (10, None), (10, [1, 3, 3, 1, 1, 1])])
def test_custom_channel_groups(cuda_lib, oracle, channels, groups):
    s = scenes.random_soup(batch=2, width=48, height=40, n_faces=50, channels=channels, seed=channels)
    check_against_oracle(oracle, s, groups=groups, label='groups %s' % groups, ids_modes=('given',))


def _bench_workloads():
    import bench
    return [(name,) + bench.WORKLOADS[name][:2] for name in sorted(bench.WORKLOADS)]


@pytest.mark.parametrize('name,gen,kwargs', _bench_workloads(), ids=[w[0] for w in _bench_workloads()])
def test_benched_workloads(cuda_lib, oracle, name, gen, kwargs):
    """cfg2, cfg3, cfg4, cfg5 and the cube as bench.py renders them, at their benched batch and frame sizes."""
    check_against_oracle(oracle, getattr(scenes, gen)(**kwargs), seed=17, label='bench ' + name, ids_modes=('given',))


@pytest.mark.parametrize('channels,groups', kp.OVERFLOW_CHANNELS)
def test_face_table_overflow_fans(cuda_lib, oracle, channels, groups):
    check_against_oracle(oracle, kp.overflow_scene(channels, 64), groups=groups, label='fans', ids_modes=('given',))


@pytest.mark.parametrize('channels,groups', kp.FLAT_ORDER_CHANNELS)
def test_flat_order_taps_across_images(cuda_lib, oracle, channels, groups):
    for W in (32, 37):
        check_against_oracle(oracle, kp.flat_order_scene(channels, W), groups=groups, label='flat order W=%d' % W,
                             ids_modes=('given',))


def test_past_the_grid_limit(cuda_lib, oracle):
    check_against_oracle(oracle, kp.grid_limit_scene(), label='B=65544', ids_modes=('given',))


@pytest.mark.parametrize('H,W', [(8, 65536), (65537, 8)])
def test_record_limit_frames(cuda_lib, oracle, H, W):
    check_against_oracle(oracle, kp.edge_strip(H, W, 3), label='%dx%d' % (H, W), ids_modes=('given',))


def _flag_reference(oracle, s, gp, flags):
    pixels_o = oracle.forward(**s)
    gb, gv, gc = oracle.backward(s['vertices'], s['faces'], pixels_o, gp)
    if flags & 1:
        gv, gc = gv.sum(0, dtype=np.float64), gc.sum(0, dtype=np.float64)
    if flags & 2:
        gv = np.zeros_like(gv)
    if flags & 4:
        gc, gb = np.zeros_like(gc), None
    return pixels_o, gb, gv, gc


@pytest.mark.parametrize('flags', FLAGS)
def test_flags_match_oracle_and_repeat_bit_for_bit(cuda_lib, oracle, flags):
    import torch
    s = scenes.config3(batch=3, width=96, height=80, level=2, background='uniform')
    t = _cuda(s)
    gp = np.random.default_rng(5).standard_normal(oracle.forward(**s).shape).astype(np.float32)
    pixels_o, gb_o, gv_o, gc_o = _flag_reference(oracle, s, gp, flags)
    pixels, gp_t = torch.from_numpy(pixels_o).cuda(), torch.from_numpy(gp).cuda()
    first = det_call(t, pixels, gp_t, None, None, flags)[:3]
    if gb_o is not None:
        np.testing.assert_array_equal(first[0].cpu().numpy(), gb_o)
    for a, b in ((first[1], gv_o), (first[2], gc_o)):
        assert rel_close(a.cpu().numpy(), b)[0]
    # eager repeat and graph replay: bit-identical
    ids = oracle.forward(**s, return_face_ids=True)[1]
    ids_t = torch.from_numpy(ids).cuda()
    eager = [x.clone() for x in det_call(t, pixels, gp_t, ids_t, None, flags)[:3]]
    again = det_call(t, pixels, gp_t, ids_t, None, flags)[:3]
    out = tuple(torch.zeros_like(x) for x in eager)
    gb, gv, gc, scratch = det_call(t, pixels, gp_t, ids_t, None, flags, out=out)   # warm-up, and the scratch to reuse
    torch.cuda.synchronize()
    for x in out:
        x.zero_()
    graph = torch.cuda.CUDAGraph()
    from dirt_b200 import rasterise_ops as ops
    ws, _ = ops._workspace(3, 80, 96, 3, t['vertices'].shape[1], t['faces'].shape[1], pixels.device)
    with torch.cuda.graph(graph):
        det_call(t, pixels, gp_t, ids_t, None, flags, ws=ws, out=out, scratch=scratch)
    for x in out:
        x.fill_(3.0)
    graph.replay()
    torch.cuda.synchronize()
    for name, a, b, c in zip(('grad_background', 'grad_vertices', 'grad_vertex_colors'), eager, again, out):
        if flags & 4 and name == 'grad_background':
            continue
        assert torch.equal(a, b), name + ': two eager calls differ'
        assert torch.equal(a, c), name + ': graph replay differs from the eager call'
    assert torch.equal(eager[1], first[1]), 'ids given and ids derived differ'


def test_item_alone_equals_item_in_batch(cuda_lib, oracle):
    import torch
    s = scenes.random_soup(batch=4, width=64, height=48, n_faces=60, channels=3, seed=21)
    pixels_o = oracle.forward(**s)
    gp = np.random.default_rng(2).standard_normal(pixels_o.shape).astype(np.float32)
    t = _cuda(s)
    _, gv, gc, _ = det_call(t, torch.from_numpy(pixels_o).cuda(), torch.from_numpy(gp).cuda())
    for b in range(4):
        one = {k: v[b:b + 1] for k, v in s.items()}
        _, gv1, gc1, _ = det_call(_cuda(one), torch.from_numpy(pixels_o[b:b + 1].copy()).cuda(),
                                  torch.from_numpy(gp[b:b + 1].copy()).cuda())
        assert torch.equal(gv[b], gv1[0]) and torch.equal(gc[b], gc1[0]), 'item %d' % b


def test_invalid_faces_and_non_finite_vertices_are_culled(cuda_lib, oracle):
    import torch
    s = scenes.random_soup(batch=2, width=56, height=40, n_faces=40, channels=3, seed=8)
    s['faces'][0, 3] = [0, 1, 10 ** 6]
    s['faces'][1, 5] = [-1, 2, 3]
    s['vertices'][1, int(s['faces'][1, 9, 0])] = [np.nan, 0.0, 0.0, 1.0]
    s['vertices'][0, int(s['faces'][0, 11, 1])] = [np.inf, 0.0, 0.0, 1.0]
    pixels_o, ids_o = oracle.forward(**s, return_face_ids=True)
    gp = np.random.default_rng(3).standard_normal(pixels_o.shape).astype(np.float32)
    t = _cuda(s)
    from dirt_b200 import rasterise_ops as ops
    default = ops.rasterise_backward_raw(t['vertices'], t['faces'], torch.from_numpy(pixels_o).cuda(),
                                         torch.from_numpy(gp).cuda(), torch.from_numpy(ids_o).cuda(), deterministic=False)
    det = det_call(t, torch.from_numpy(pixels_o).cuda(), torch.from_numpy(gp).cuda(), torch.from_numpy(ids_o).cuda())
    assert torch.equal(default[0], det[0])
    for a, b in ((det[1], default[1]), (det[2], default[2])):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        np.testing.assert_array_equal(np.isfinite(a), np.isfinite(b))
        assert rel_close(np.nan_to_num(a), np.nan_to_num(b))[0]


@pytest.fixture
def deterministic_algorithms():
    import torch
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)


def test_public_api_follows_torch_deterministic_algorithms(cuda_lib, oracle, deterministic_algorithms):
    import torch
    import dirt_b200 as dirt
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=3, width=128, height=96, level=2, background='uniform')
    gp = torch.from_numpy(np.random.default_rng(7).standard_normal((3, 96, 128, 4)).astype(np.float32)).cuda()
    grads = []
    for _ in range(2):
        t = _cuda(s)
        for k in ('background', 'vertices', 'vertex_colors'):
            t[k].requires_grad_(True)
        pixels = dirt.rasterise_batch(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
        (pixels * gp).sum().backward()
        grads.append([t[k].grad.clone() for k in ('background', 'vertices', 'vertex_colors')])
    for a, b in zip(*grads):
        assert torch.equal(a, b)
    t = _cuda(s)
    raw = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels.detach(), gp, None, [3, 1], deterministic=True)
    assert torch.equal(grads[0][0], raw[0]) and torch.equal(grads[0][1], raw[1]) and torch.equal(grads[0][2], raw[2])
    default = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels.detach(), gp, None, [3, 1], deterministic=False)
    for a, b in zip(raw, default):
        assert rel_close(a.cpu().numpy(), b.cpu().numpy())[0]


def test_deferred_public_api_follows_torch_deterministic_algorithms(cuda_lib, deterministic_algorithms):
    import torch
    import dirt_b200 as dirt
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=2, width=128, height=96, level=2, background='uniform')
    t = _cuda(s)
    attrs = torch.cat([t['vertex_colors'][..., :3], t['vertices'][..., :3]], dim=-1).contiguous()
    bg = torch.zeros(2, 96, 128, 6, device='cuda')

    def shader(g):
        return torch.sigmoid(g[..., :3] * 2.0 + g[..., 3:6])

    runs = []
    for _ in range(2):
        v = t['vertices'].clone().requires_grad_(True)
        a = attrs.clone().requires_grad_(True)
        out = dirt.rasterise_batch_deferred(bg, v, a, t['faces'], shader)
        (out ** 2).sum().backward()
        runs.append((v.grad.clone(), a.grad.clone(), out.detach()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    pixels = runs[0][2]
    _, gv, _ = ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, 2 * pixels, None, [3], deterministic=True,
                                          want_colour=False)
    assert torch.equal(gv, runs[0][0])
