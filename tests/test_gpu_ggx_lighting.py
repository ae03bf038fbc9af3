"""GPU: the GGX specular model's CUDA path (`lighting.specular_ggx_directional`, `specular_ggx_point`) against its torch
restatement (`lighting._specular_ggx`).

Forward values and every gradient against the float64 restatement and float64 autograd (conftest.rel_close, 1e-4).
Random inputs keep |n . l| and |n . v| >= 1e-3, away from the jump of the gradient at the mask; the mask's boundary is
tested with exact values.  The parameter gradients are summed in a fixed order: repeats, graph replays and an item
alone or inside a batch give bit-identical results."""
import math

import numpy as np
import pytest
import torch

from conftest import rel_close

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
KEYS = ['pos', 'nrm', 'rough', 'spec', 'light', 'lcol', 'cam']
PARAMS = ['light', 'lcol', 'cam']


@pytest.fixture(scope='module')
def lighting(cuda_lib):
    from dirt_b200 import lighting
    return lighting


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _unit(x):
    return torch.nn.functional.normalize(x, dim=-1)


def _away_from_the_mask(x, point, g):
    """Re-draws the normals whose |n . l| or |n . v| (in float64) is below 1e-3."""
    for _ in range(20):
        p, n = x['pos'].double(), _unit(x['nrm'].double())
        light = x['light'].double()[..., None, :]
        l = _unit(light - p) if point else _unit(-light).expand_as(p)
        v = _unit(x['cam'].double()[..., None, :] - p)
        bad = (((n * l).sum(-1).abs() < 1e-3) | ((n * v).sum(-1).abs() < 1e-3))
        if not bad.any():
            return x
        fresh = torch.randn(x['nrm'].shape, generator=g, device=DEV)
        x['nrm'] = torch.where(bad[..., None], fresh, x['nrm'])
    raise AssertionError('could not draw normals away from the mask')


def _inputs(seed, point, lead=(), V=3000, C=3, per_item=False):
    """Positions in a 4-unit box, normals of random length, the camera and a point light outside the box, roughness in
    [0.02, 1) (some below the clamp at 0.045), F0 in [0, 1)."""
    g = _gen(seed)
    item = lead if per_item else ()
    x = dict(pos=torch.rand(lead + (V, 3), generator=g, device=DEV) * 4 - 2,
             nrm=torch.randn(lead + (V, 3), generator=g, device=DEV),
             rough=torch.rand(lead + (V, 1), generator=g, device=DEV) * 0.98 + 0.02,
             spec=torch.rand(lead + (V, C), generator=g, device=DEV),
             light=(torch.randn(item + (3,), generator=g, device=DEV) * 3 + 4) if point else
             _unit(torch.randn(item + (3,), generator=g, device=DEV)),
             lcol=torch.rand(item + (C,), generator=g, device=DEV) + 0.5,
             cam=torch.randn(item + (3,), generator=g, device=DEV) + torch.tensor([0., 0., 6.], device=DEV))
    return _away_from_the_mask(x, point, g)


def _op(lighting, point, x, ds):
    fn = lighting.specular_ggx_point if point else lighting.specular_ggx_directional
    return fn(*[x[k] for k in KEYS], double_sided=ds)


def _ref(lighting, point, x, ds):
    return lighting._specular_ggx(*[x[k] for k in KEYS], point, ds)


def _check_forward(lighting, point, x, ds, tag):
    got = _op(lighting, point, x, ds)
    want = _ref(lighting, point, {k: v.double() for k, v in x.items()}, ds)
    assert got.shape == want.shape and got.dtype == torch.float32, tag
    ok, ratio = rel_close(got.cpu().numpy(), want.cpu().numpy(), name='ggx fwd')
    assert ok, (tag, point, ds, ratio)
    return got


def _grads_of(fn, x, keys, grad_out):
    leaves = {k: v.detach().clone().requires_grad_(k in keys) for k, v in x.items()}
    (fn(leaves) * grad_out).sum().backward()
    return {k: leaves[k].grad for k in keys}


def _check_grads(lighting, point, x, ds, keys, seed, tag):
    """grad_out in [0.5, 1.5) (a mean-like loss), so that the parameter gradients' sums over the points are not far
    smaller than their terms."""
    out_shape = _op(lighting, point, x, ds).shape
    grad_out = torch.rand(out_shape, generator=_gen(seed), device=DEV) + 0.5
    got = _grads_of(lambda l: _op(lighting, point, l, ds), x, keys, grad_out)
    want = _grads_of(lambda l: _ref(lighting, point, {k: v.double() for k, v in l.items()}, ds), x, keys,
                     grad_out.double())
    for k in keys:
        assert got[k] is not None and got[k].shape == x[k].shape, (tag, k)
        ok, ratio = rel_close(got[k].cpu().numpy(), want[k].cpu().numpy(), name='ggx grad %s' % k)
        assert ok, (tag, point, ds, k, ratio)


CASES = [((), 5000, False, 'no batch'), ((3,), 1000, True, 'per item'), ((2, 2), 700, False, 'rank 2, shared')]


@pytest.mark.parametrize('C', [1, 3, 4, 5])
@pytest.mark.parametrize('ds', [False, True])
@pytest.mark.parametrize('point', [False, True])
def test_forward_and_gradients_match_the_restatement(lighting, point, ds, C):
    for i, (lead, V, per_item, tag) in enumerate(CASES):
        x = _inputs(100 * C + 10 * i + 2 * point + ds, point, lead, V, C, per_item)
        _check_forward(lighting, point, x, ds, tag)
        _check_grads(lighting, point, x, ds, KEYS, 7 + i, tag)


def _highlights(seed, point, a_max, V=4000, C=3):
    """Points inside sharp highlights: the normal within a few a^2 of the half vector, roughness in [0.03, a_max)
    (the clamp included), where D and its gradient change fastest."""
    g = _gen(seed)
    x = _inputs(seed, point, (), V, C)
    x['rough'] = torch.rand(V, 1, generator=g, device=DEV) * (a_max - 0.03) + 0.03
    p = x['pos'].double()
    l = _unit(x['light'].double() - p) if point else _unit(-x['light'].double()).expand_as(p)
    h = _unit(l + _unit(x['cam'].double() - p))
    a2 = x['rough'].double().clamp(min=0.045) ** 2
    x['nrm'] = (_unit(h + torch.randn(V, 3, generator=g, device=DEV, dtype=torch.float64) * a2 * 2) *
                (torch.rand(V, 1, generator=g, device=DEV, dtype=torch.float64) + 0.5)).float()
    return _away_from_the_mask(x, point, g)


@pytest.mark.parametrize('point', [False, True])
def test_sharp_highlights_down_to_the_clamp(lighting, point):
    for a_max, seed in ((0.06, 40), (0.2, 41)):
        x = _highlights(seed + 2 * point, point, a_max)
        for ds in (False, True):
            _check_forward(lighting, point, x, ds, 'highlights < %g' % a_max)
            _check_grads(lighting, point, x, ds, KEYS, 42, 'highlights < %g' % a_max)


@pytest.mark.parametrize('point', [False, True])
def test_each_needs_input_grad_alone(lighting, point):
    x = _inputs(50 + point, point, (2,), 2000, 3, per_item=True)
    for k in KEYS:
        _check_grads(lighting, point, x, False, [k], 11, 'only ' + k)


@pytest.mark.parametrize('ds', [False, True])
@pytest.mark.parametrize('point', [False, True])
def test_the_mask_and_the_clamp_at_exact_values(lighting, point, ds):
    """n . l = 0, n . v = 0, both negative, l = -v (h = 0) and a normal of length 0 give exactly 0 and zero gradients;
    roughness below 0.045 gets no gradient, roughness at exactly 0.045 (in float32) the full one."""
    f = lambda v: torch.tensor(v, device=DEV)
    pos = torch.zeros(7, 3, device=DEV)
    nrm = f([[0., 0., 1.], [0., 0., 1.], [0., 0., 1.], [0., 0., 1.], [0., 0., 0.], [0., 0.3, 1.], [0., 0.3, 1.]])
    l_dirs = f([[1., 0., 0.], [0., 0.6, 0.8], [0.6, 0., -0.8], [0.6, 0., 0.8], [0., 0.6, 0.8], [0., 0.6, 0.8],
                [0., 0.6, 0.8]])
    v_dirs = f([[0., 0.6, 0.8], [1., 0., 0.], [0., -0.6, 0.8], [-0.6, 0., -0.8], [0.6, 0., 0.8], [0.6, 0., 0.8],
                [0.6, 0., 0.8]])
    rough = f([[0.3], [0.3], [0.3], [0.3], [0.3], [0.03], [0.045]])
    for i in range(7):   # one point per call: the light and the camera belong to it
        x = dict(pos=pos[i:i + 1], nrm=nrm[i:i + 1], rough=rough[i:i + 1], spec=f([[0.5, 0.2]]),
                 light=(2 * l_dirs[i]) if point else -l_dirs[i], lcol=f([1., 2.]), cam=3 * v_dirs[i])
        got = _op(lighting, point, x, ds)
        grads = _grads_of(lambda l: _op(lighting, point, l, ds), x, KEYS, torch.ones_like(got))
        want = _grads_of(lambda l: _ref(lighting, point, {k: v.double() for k, v in l.items()}, ds), x, KEYS,
                         torch.ones_like(got).double())
        if i < 5:
            assert torch.equal(got, torch.zeros_like(got)), i
            for k in KEYS:
                assert torch.equal(grads[k], torch.zeros_like(grads[k])), (i, k)
                assert torch.equal(want[k], torch.zeros_like(want[k])), (i, k)
            continue
        assert (got > 0).all(), i
        if i == 5:
            assert torch.equal(grads['rough'], torch.zeros_like(grads['rough']))
        else:
            assert float(grads['rough'].abs()) > 0
        for k in KEYS:
            ok, ratio = rel_close(grads[k].cpu().numpy(), want[k].cpu().numpy(), name='ggx grad at the clamp')
            assert ok, (i, k, ratio)


def test_strided_gbuffer_slices_go_in_without_a_copy(lighting):
    from dirt_b200.lighting import _rows
    g = _gen(12)
    B, H, W = 2, 64, 48
    gbuffer = torch.rand(B, H, W, 12, generator=g, device=DEV)
    gbuffer[..., 0:3] = gbuffer[..., 0:3] * 4 - 2
    gbuffer[..., 3:6] = _unit(gbuffer[..., 3:6] - 0.5 + torch.tensor([0., 0., 0.6], device=DEV))
    pos, nrm, spec = (gbuffer[..., a:b].reshape(B, -1, 3) for a, b in ((0, 3), (3, 6), (7, 10)))
    rough = gbuffer[..., 6:7].reshape(B, -1, 1)
    for t, k in ((pos, 3), (nrm, 3), (spec, 3), (rough, 1)):
        assert _rows(t, k).data_ptr() == t.data_ptr() and _rows(t, k).stride(0) == 12
    for point in (False, True):
        light = torch.tensor([1., 2., 5.], device=DEV) if point else _unit(torch.tensor([0.3, -0.2, -1.], device=DEV))
        x = dict(pos=pos, nrm=nrm, rough=rough, spec=spec, light=light, lcol=torch.ones(3, device=DEV),
                 cam=torch.tensor([0., 1., 6.], device=DEV))
        x = _away_from_the_mask(x, point, g)
        for ds in (False, True):
            _check_forward(lighting, point, x, ds, 'gbuffer slices')
            _check_grads(lighting, point, x, ds, KEYS, 13, 'gbuffer slices')


def test_empty_inputs(lighting):
    for point in (False, True):
        for lead, V, per_item in (((), 0, False), ((0,), 50, True), ((0,), 50, False), ((3,), 0, True)):
            x = {k: v.requires_grad_(True) for k, v in _inputs(16, point, lead, V, 3, per_item).items()}
            out = _op(lighting, point, x, False)
            assert out.shape == lead + (V, 3)
            out.sum().backward()
            for k in KEYS:
                assert x[k].grad is not None and x[k].grad.shape == x[k].shape and not x[k].grad.any(), (lead, V, k)


@pytest.mark.parametrize('point', [False, True])
def test_double_backward(lighting, point):
    x = _inputs(20 + point, point, (2,), 300, 3, per_item=True)
    grad_out = torch.randn(_op(lighting, point, x, False).shape, generator=_gen(21), device=DEV)

    def second(fn):
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in x.items()}
        first = torch.autograd.grad((fn(leaves) * grad_out).sum(), [leaves[k] for k in KEYS], create_graph=True)
        sum(g.square().sum() for g in first).backward()
        return first, [leaves[k].grad for k in KEYS]

    first_op, second_op = second(lambda l: _op(lighting, point, l, False))
    first_ref, second_ref = second(lambda l: _ref(lighting, point, l, False))
    for k, a, b in zip(KEYS * 2, first_op + tuple(second_op), first_ref + tuple(second_ref)):
        ok, ratio = rel_close(a.detach().cpu().numpy(), b.detach().cpu().numpy(), name='ggx double backward')
        assert ok, (point, k, ratio)
    # gradcheck-style: the first gradient's own gradient against finite differences, in float64 through the op's
    # create_graph path (the restatement)
    leaves = {k: v.detach()[:1, :5].double().clone().requires_grad_(True) if k in ('pos', 'nrm', 'rough', 'spec')
              else v.detach()[:1].double().clone().requires_grad_(True) for k, v in x.items()}
    assert torch.autograd.gradgradcheck(lambda *t: _ref(lighting, point, dict(zip(KEYS, t)), False),
                                        [leaves[k] for k in KEYS])


@pytest.mark.parametrize('per_item', [True, False])
def test_parameter_gradients_are_deterministic(lighting, per_item):
    for point in (False, True):
        x = _inputs(22 + point, point, (4,), 100000, 3, per_item)
        grad_out = torch.randn(_op(lighting, point, x, True).shape, generator=_gen(23), device=DEV)
        runs = [_grads_of(lambda l: _op(lighting, point, l, True), x, KEYS, grad_out) for _ in range(3)]
        for k in KEYS:
            assert all(torch.equal(r[k].view(torch.int32), runs[0][k].view(torch.int32)) for r in runs[1:]), k


@pytest.mark.parametrize('C', [3, 2])
def test_an_item_alone_and_inside_a_batch_give_identical_gradients(lighting, C):
    for point in (False, True):
        x = _inputs(26 + point, point, (5,), 5000, C, per_item=True)
        grad_out = torch.randn(_op(lighting, point, x, False).shape, generator=_gen(27), device=DEV)
        batch = _grads_of(lambda l: _op(lighting, point, l, False), x, KEYS, grad_out)
        for b in (0, 3):
            alone = {k: v[b] for k, v in x.items()}   # no batch, its parameters shared
            single = _grads_of(lambda l: _op(lighting, point, l, False), alone, KEYS, grad_out[b])
            for k in KEYS:
                assert torch.equal(single[k].view(torch.int32), batch[k][b].view(torch.int32)), (point, b, k)


@pytest.mark.parametrize('point', [False, True])
def test_cuda_graph_capture_and_replay(lighting, point):
    x = {k: v.requires_grad_(True) for k, v in _inputs(28 + point, point, (2,), 50000, 3).items()}
    grad_out = torch.randn(_op(lighting, point, x, False).shape, generator=_gen(29), device=DEV)

    def step():
        for v in x.values():
            v.grad = None
        out = _op(lighting, point, x, False)
        (out * grad_out).sum().backward()
        return out

    eager = step().detach().clone()
    eager_grads = {k: x[k].grad.clone() for k in KEYS}
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
        for k in KEYS:
            assert torch.equal(x[k].grad, eager_grads[k]), k


# ---- through the deferred rasteriser ---------------------------------------------------------------------------------

def _sphere_scene(batch, size, seed):
    """cfg3's posed icosphere-4 batch with G-buffer attributes [mask, albedo rgb, normal xyz] per vertex.  The spheres
    are unit spheres about their centres, so the normal is also the shaded point's position in the sphere's frame."""
    from dirt_b200 import scenes
    s = scenes.config3(batch=batch, width=size, height=size, seed=seed)
    attrs = torch.from_numpy(s['vertex_colors']).to(DEV)                        # [B, V, 4]: mask, unit normal
    albedo = torch.rand(attrs.shape[:2] + (3,), generator=_gen(seed), device=DEV) * 0.6 + 0.2
    attributes = torch.cat([attrs[..., :1], albedo, attrs[..., 1:]], -1)        # [B, V, 7]
    background = torch.zeros(batch, size, size, 7, device=DEV)
    return (background, torch.from_numpy(s['vertices']).to(DEV), attributes, torch.from_numpy(s['faces']).to(DEV))


LIGHTS = [(-0.3, -0.4, -1.), (0.8, 0.2, -0.6), (-0.5, 0.7, -0.5)]   # directions the light travels along
CAMERA = (0., 0., 4.)


def _shader(diffuse, ggx, lights=LIGHTS):
    """Diffuse plus GGX under directional lights, from per-pixel roughness [B, H, W, 1] and specular colour
    [B, H, W, 3], blended with a black background by the mask."""
    def shader_fn(gbuffer, roughness, specular):
        B, H, W, _ = gbuffer.shape
        mask, albedo, normals = gbuffer[..., :1], gbuffer[..., 1:4].reshape(B, -1, 3), gbuffer[..., 4:7].reshape(B, -1, 3)
        lit = 0.
        for d in lights:
            d = _unit(torch.tensor(d, device=DEV))
            colour = torch.ones(3, device=DEV)
            lit = lit + diffuse(normals, albedo, d, colour, double_sided=False) + ggx(
                normals, normals, roughness.reshape(B, -1, 1), specular.reshape(B, -1, 3), d, colour,
                torch.tensor(CAMERA, device=DEV))
        return lit.reshape(B, H, W, 3) * mask
    return shader_fn


def _restatement_fp64(vertex_positions, vertex_normals, vertex_roughness, vertex_specular, light_direction,
                      light_color, camera_position, double_sided=False, name=None):
    from dirt_b200 import lighting
    return lighting._specular_ggx(vertex_positions.double(), vertex_normals.double(), vertex_roughness.double(),
                                  vertex_specular.double(), light_direction.double(), light_color.double(),
                                  camera_position.double(), False, double_sided).float()


def test_deferred_diffuse_plus_ggx_through_rasterise_batch_deferred(lighting):
    """A cfg3-sized batch (64 x 512^2) under one light: finite gradients to the vertices, the attributes and the
    material maps, and pixels and material gradients that match the same shader with the float64 restatement in the
    op's place."""
    import dirt_b200 as dirt
    background, vertices, attributes, faces = _sphere_scene(64, 512, 1)
    g = _gen(2)
    rough0 = torch.rand(64, 512, 512, 1, generator=g, device=DEV) * 0.8 + 0.1
    spec0 = torch.rand(64, 512, 512, 3, generator=g, device=DEV) * 0.5
    weights = torch.rand(64, 512, 512, 3, generator=g, device=DEV)

    def run(ggx):
        v, a, r, s = (t.clone().requires_grad_(True) for t in (vertices, attributes, rough0, spec0))
        pixels = dirt.rasterise_batch_deferred(background, v, a, faces,
                                               _shader(lighting.diffuse_directional, ggx, LIGHTS[:1]), [r, s])
        (pixels * weights).sum().backward()
        return pixels.detach(), v.grad, a.grad, r.grad, s.grad

    op = run(lighting.specular_ggx_directional)
    assert float((op[0] != 0).any(-1).float().mean()) > 0.2   # the spheres are in view
    for name, t in zip(('vertices', 'attributes', 'roughness', 'specular'), op[1:]):
        assert t is not None and torch.isfinite(t).all(), name
        assert t.abs().sum() > 0, name
    ref = run(_restatement_fp64)
    ok, ratio = rel_close(op[0].cpu().numpy(), ref[0].cpu().numpy(), name='ggx deferred pixels')
    assert ok, ratio
    for name, a, b in zip(('roughness', 'specular'), op[3:], ref[3:]):
        ok, ratio = rel_close(a.cpu().numpy(), b.cpu().numpy(), name='ggx deferred grad_' + name)
        assert ok, (name, ratio)


FIT_STEPS = 100
FIT_RATIO = 1000   # chosen on an H100 (80GB HBM3, 700 W): the loss fell 29 000x in 100 steps, 16x in 25, 232x in 50


def test_fitting_roughness_and_specular_colour_through_the_rasteriser(lighting):
    """Images rendered with known per-pixel roughness and specular colour; both fitted from a uniform start with Adam
    through rasterise_batch_deferred at 4 x 128^2.  The masked MSE must fall at least FIT_RATIO x in FIT_STEPS steps."""
    import dirt_b200 as dirt
    B, size = 4, 128
    background, vertices, attributes, faces = _sphere_scene(B, size, 4)
    shader = _shader(lighting.diffuse_directional, lighting.specular_ggx_directional)
    g = _gen(5)
    truth_r = torch.rand(B, size, size, 1, generator=g, device=DEV) * 0.5 + 0.15
    truth_s = torch.rand(B, size, size, 3, generator=g, device=DEV) * 0.6 + 0.2
    with torch.no_grad():
        target = dirt.rasterise_batch_deferred(background, vertices, attributes, faces, shader, [truth_r, truth_s])
        mask = dirt.rasterise_batch_deferred(background, vertices, attributes, faces,
                                             lambda gb, r, s: gb[..., :1].expand(-1, -1, -1, 3), [truth_r, truth_s])
    assert float(mask.mean()) > 0.2
    rough = torch.full((B, size, size, 1), 0.5, device=DEV, requires_grad=True)
    spec = torch.full((B, size, size, 3), 0.5, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([rough, spec], lr=0.02)
    losses = []
    for step in range(FIT_STEPS):
        opt.zero_grad()
        pixels = dirt.rasterise_batch_deferred(background, vertices, attributes, faces, shader, [rough, spec])
        loss = (((pixels - target) * mask) ** 2).sum() / mask.sum()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    ratio = losses[0] / losses[-1]
    print('ggx fit: loss %.3e -> %.3e (ratio %.1f) after %d steps; at 25/50/75: %s' % (
        losses[0], losses[-1], ratio, FIT_STEPS, [round(losses[0] / losses[k - 1], 1) for k in (25, 50, 75)]))
    assert ratio >= FIT_RATIO, ratio
