"""GPU: the reflectance models' CUDA path against their torch restatement (the private functions of
dirt_b200/lighting.py).

Forward values against the restatement in float64 and in float32 on the same device, at the tolerance
test_helpers_cpu.test_reflectance_models_match_the_loop_restatements grants the restatement itself (atol 2e-6; rtol 2e-4
for the specular model).  Gradients against float64 autograd of the restatement with conftest.rel_close (1e-4)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import rel_close

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device('cuda', 0)
MODELS = ['diffuse_directional', 'specular_directional', 'diffuse_point']
ARGS = {'diffuse_directional': ['nrm', 'col', 'ldir', 'lcol'],
        'specular_directional': ['pos', 'nrm', 'col', 'ldir', 'lcol', 'cam', 'shin'],
        'diffuse_point': ['pos', 'nrm', 'col', 'lpos', 'lcol']}
PER_POINT = {'pos', 'nrm', 'col'}


@pytest.fixture(scope='module')
def lighting(cuda_lib):
    from dirt_b200 import lighting
    return lighting


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _inputs(seed, lead=(), V=3000, C=3, per_item=False):
    """Unit normals, positions in a 4-unit box, a camera and a point light outside it, shininess in [1, 9)."""
    g = _gen(seed)
    item = lead if per_item else ()
    n = torch.nn.functional.normalize(torch.randn(lead + (V, 3), generator=g, device=DEV), dim=-1)
    return dict(pos=torch.rand(lead + (V, 3), generator=g, device=DEV) * 4 - 2, nrm=n,
                col=torch.rand(lead + (V, C), generator=g, device=DEV),
                ldir=torch.nn.functional.normalize(torch.randn(item + (3,), generator=g, device=DEV), dim=-1),
                lcol=torch.rand(item + (C,), generator=g, device=DEV) + 0.5,
                lpos=torch.randn(item + (3,), generator=g, device=DEV) * 3 + 4,
                cam=torch.randn(item + (3,), generator=g, device=DEV) + torch.tensor([0., 0., 6.], device=DEV),
                shin=torch.rand(item, generator=g, device=DEV) * 8 + 1)


def _op(lighting, model, x, ds):
    return getattr(lighting, model)(*[x[k] for k in ARGS[model]], double_sided=ds)


def _ref(lighting, model, x, ds):
    return getattr(lighting, '_' + model)(*[x[k] for k in ARGS[model]], double_sided=ds)


def _check_forward(lighting, model, x, ds, tag):
    got = _op(lighting, model, x, ds)
    rtol = 2e-4 if model == 'specular_directional' else 1e-7
    for label, want in (('fp64', _ref(lighting, model, {k: v.double() for k, v in x.items()}, ds)),
                        ('fp32', _ref(lighting, model, x, ds))):
        want = want.float()
        assert got.shape == want.shape and got.dtype == torch.float32
        a, b = got.cpu().numpy(), want.cpu().numpy()
        rel_close(a, b, rel=2e-4 if rtol > 1e-6 else 1e-4, name='lighting %s fwd vs %s' % (model, label))
        np.testing.assert_allclose(a, b, rtol=rtol, atol=2e-6, err_msg='%s %s vs %s' % (tag, model, label))
    return got


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
@pytest.mark.parametrize('ds', [True, False])
@pytest.mark.parametrize('model', MODELS)
def test_forward_matches_the_restatement(lighting, model, ds, C):
    _check_forward(lighting, model, _inputs(1, (), 5000, C), ds, 'no batch')
    _check_forward(lighting, model, _inputs(2, (3,), 1000, C, per_item=True), ds, 'per item')
    _check_forward(lighting, model, _inputs(3, (2, 2), 700, C), ds, 'shared')


def _grads_of(fn, x, keys, grad_out):
    leaves = {k: v.detach().clone().requires_grad_(k in keys) for k, v in x.items()}
    (fn(leaves) * grad_out).sum().backward()
    return {k: leaves[k].grad for k in keys}


def _check_grads(lighting, model, x, ds, keys, seed, tag):
    """grad_out in [0.5, 1.5) (a mean-like loss).  Near the highlight's centre the shininess gradient's log(t) has few
    correct bits in any fp32 evaluation; under a random-sign grad_out the sum over the points can be far smaller than its
    terms, and that rounding would then be measured against the small sum instead of against the terms."""
    out_shape = _op(lighting, model, x, ds).shape
    grad_out = torch.rand(out_shape, generator=_gen(seed), device=DEV) + 0.5
    got = _grads_of(lambda l: _op(lighting, model, l, ds), x, keys, grad_out)
    want = _grads_of(lambda l: _ref(lighting, model, {k: v.double() for k, v in l.items()}, ds), x, keys,
                     grad_out.double())
    for k in keys:
        assert got[k] is not None and got[k].shape == x[k].shape, (tag, k)
        ok, ratio = rel_close(got[k].cpu().numpy(), want[k].cpu().numpy(), name='lighting %s grad %s' % (model, k))
        assert ok, (tag, model, ds, k, ratio)


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5])
@pytest.mark.parametrize('ds', [True, False])
@pytest.mark.parametrize('model', MODELS)
def test_gradients_match_autograd_of_the_restatement(lighting, model, ds, C):
    keys = ARGS[model]
    _check_grads(lighting, model, _inputs(4, (), 3000, C), ds, keys, 5, 'no batch')
    _check_grads(lighting, model, _inputs(6, (3,), 1000, C, per_item=True), ds, keys, 7, 'per item')
    _check_grads(lighting, model, _inputs(8, (2, 2), 600, C), ds, keys, 9, 'shared')


@pytest.mark.parametrize('model', MODELS)
def test_each_needs_input_grad_alone(lighting, model):
    x = _inputs(10, (2,), 2000, 3, per_item=True)
    for k in ARGS[model]:
        _check_grads(lighting, model, x, False, [k], 11, 'only ' + k)


def test_strided_gbuffer_slices_go_in_without_a_copy(lighting):
    from dirt_b200.lighting import _rows
    g = _gen(12)
    gbuffer = torch.rand(2, 64, 48, 10, generator=g, device=DEV)
    gbuffer[..., 7:] = torch.nn.functional.normalize(gbuffer[..., 7:] - 0.5, dim=-1)
    pos, col, nrm = (gbuffer[..., a:b].reshape(-1, 3) for a, b in ((1, 4), (4, 7), (7, 10)))
    assert _rows(nrm, 3).data_ptr() == nrm.data_ptr() and _rows(nrm, 3).stride() == (10, 1)
    x = dict(pos=pos, nrm=nrm, col=col, ldir=torch.tensor([0.6, -0.8, 0.], device=DEV), lcol=torch.ones(3, device=DEV),
             lpos=torch.tensor([1., 2., 3.], device=DEV), cam=torch.tensor([0., 0., 5.], device=DEV),
             shin=torch.tensor(6., device=DEV))
    for model in MODELS:
        for ds in (True, False):
            _check_forward(lighting, model, x, ds, 'gbuffer slices')
            _check_grads(lighting, model, x, ds, ARGS[model], 13, 'gbuffer slices')
    # a transposed (non-unit last stride) and an expanded input are handled too
    y = _inputs(14, (), 500, 3)
    y['nrm'] = y['nrm'].t().contiguous().t()
    y['col'] = y['col'][:1].expand(500, 3)
    for model in MODELS:
        _check_forward(lighting, model, y, False, 'transposed / expanded')
        _check_grads(lighting, model, y, False, ARGS[model], 15, 'transposed / expanded')


@pytest.mark.parametrize('model', MODELS)
def test_empty_inputs(lighting, model):
    for lead, V, per_item in (((), 0, False), ((0,), 50, True), ((0,), 50, False), ((3,), 0, True)):
        x = {k: v.requires_grad_(True) for k, v in _inputs(16, lead, V, 3, per_item).items()}
        out = _op(lighting, model, x, True)
        assert out.shape == lead + (V, 3)
        out.sum().backward()
        for k in ARGS[model]:
            assert x[k].grad is not None and x[k].grad.shape == x[k].shape and not x[k].grad.any(), (lead, V, k)


def _kink_inputs():
    """Points exactly at the kinks: cosine exactly 0 (normal perpendicular to the light), negative cosines (term 0), a
    point at the light position (zero vector's norm)."""
    nrm = torch.tensor([[1., 0., 0.], [0., 0., 1.], [0., 1., 0.], [0., -1., 0.], [0.6, 0.8, 0.]], device=DEV)
    pos = torch.tensor([[1., 2., 3.], [0., 0., 0.], [1., 0., 0.], [0.5, 0.5, 0.5], [2., 1., 0.]], device=DEV)
    return dict(nrm=nrm, pos=pos, col=torch.full((5, 3), 0.5, device=DEV), ldir=torch.tensor([0., 1., 0.], device=DEV),
                lcol=torch.tensor([1., 0.5, 0.25], device=DEV), lpos=torch.tensor([1., 2., 3.], device=DEV),
                cam=torch.tensor([0., 5., 0.], device=DEV), shin=torch.tensor(3., device=DEV))


@pytest.mark.parametrize('ds', [True, False])
def test_kinks(lighting, ds):
    x = _kink_inputs()
    for model in MODELS:
        _check_forward(lighting, model, x, ds, 'kinks')
        _check_grads(lighting, model, x, ds, ARGS[model], 17, 'kinks')
    # pow's masks: exponent 0, and base 0 with exponent >= 0 (single-sided, cosine < 0 -> term 0)
    for s in (0., 1., 3.):
        y = dict(x, shin=torch.tensor(s, device=DEV))
        _check_forward(lighting, 'specular_directional', y, ds, 'pow s=%g' % s)
        _check_grads(lighting, 'specular_directional', y, ds, ARGS['specular_directional'], 18, 'pow s=%g' % s)


def test_a_point_at_the_camera_gives_nan(lighting):
    x = _inputs(19, (), 64, 3)
    x['pos'][5] = x['cam']
    got = _op(lighting, 'specular_directional', x, True)
    want = _ref(lighting, 'specular_directional', x, True)
    assert torch.isnan(got[5]).all() and torch.isnan(want[5]).all()
    keep = torch.ones(64, dtype=torch.bool, device=DEV)
    keep[5] = False
    np.testing.assert_allclose(got[keep].cpu().numpy(), want[keep].cpu().numpy(), rtol=2e-4, atol=2e-6)


@pytest.mark.parametrize('model', MODELS)
def test_double_backward(lighting, model):
    x = _inputs(20, (2,), 300, 3, per_item=True)
    keys = ARGS[model]
    grad_out = torch.randn(_op(lighting, model, x, False).shape, generator=_gen(21), device=DEV)

    def second(fn):
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in x.items()}
        first = torch.autograd.grad((fn(leaves) * grad_out).sum(), [leaves[k] for k in keys], create_graph=True)
        sum(g.square().sum() for g in first).backward()
        return first, [leaves[k].grad for k in keys]

    first_op, second_op = second(lambda l: _op(lighting, model, l, False))
    first_ref, second_ref = second(lambda l: _ref(lighting, model, l, False))
    for k, a, b in zip(keys, first_op + tuple(second_op), first_ref + tuple(second_ref)):
        ok, ratio = rel_close(a.detach().cpu().numpy(), b.detach().cpu().numpy(), name='lighting double backward')
        assert ok, (model, k, ratio)


@pytest.mark.parametrize('model', MODELS)
def test_parameter_gradients_are_deterministic(lighting, model):
    x = _inputs(22, (4,), 100000, 3)
    params = [k for k in ARGS[model] if k not in PER_POINT]
    grad_out = torch.randn(_op(lighting, model, x, True).shape, generator=_gen(23), device=DEV)
    runs = [_grads_of(lambda l: _op(lighting, model, l, True), x, params, grad_out) for _ in range(3)]
    for k in params:
        assert all(torch.equal(r[k].view(torch.int32), runs[0][k].view(torch.int32)) for r in runs[1:]), k


@pytest.mark.parametrize('model', MODELS)
def test_cuda_graph_capture_and_replay(lighting, model):
    x = {k: v.requires_grad_(True) for k, v in _inputs(24, (2,), 50000, 3).items()}
    grad_out = torch.randn(_op(lighting, model, x, False).shape, generator=_gen(25), device=DEV)

    def step():
        for v in x.values():
            v.grad = None
        out = _op(lighting, model, x, False)
        (out * grad_out).sum().backward()
        return out

    eager = step().detach().clone()
    eager_grads = {k: x[k].grad.clone() for k in ARGS[model]}
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
        for k in ARGS[model]:
            assert torch.equal(x[k].grad, eager_grads[k]), k


# ---- the deferred example's shader ---------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def deferred(cuda_lib):
    spec = importlib.util.spec_from_file_location('deferred_example', os.path.join(ROOT, 'examples', 'deferred.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _torch_diffuse_directional(vertex_normals, vertex_colors, light_direction, light_color, double_sided=True, name=None):
    from dirt_b200 import lighting
    f = lambda t: torch.as_tensor(t, dtype=torch.float32, device=vertex_normals.device)
    return lighting._diffuse_directional(f(vertex_normals), f(vertex_colors), f(light_direction), f(light_color),
                                         double_sided)


def _torch_specular_directional(vertex_positions, vertex_normals, vertex_reflectivities, light_direction, light_color,
                                camera_position, shininess, double_sided=True, name=None):
    from dirt_b200 import lighting
    f = lambda t: torch.as_tensor(t, dtype=torch.float32, device=vertex_positions.device)
    return lighting._specular_directional(f(vertex_positions), f(vertex_normals), f(vertex_reflectivities),
                                          f(light_direction), f(light_color), f(camera_position), f(shininess),
                                          double_sided)


def _with_restatement(monkeypatch, fn):
    from dirt_b200 import lighting
    with monkeypatch.context() as m:
        m.setattr(lighting, 'diffuse_directional', _torch_diffuse_directional)
        m.setattr(lighting, 'specular_directional', _torch_specular_directional)
        return fn()


def test_deferred_shader_on_a_cfg3_sized_gbuffer(deferred, monkeypatch):
    """64 x 512^2 pixels; pixels and the gradients to the G-buffer and to the light direction.  Pixels whose float64
    diffuse cosine, or whose lit value before the final clamp to [0, 1], lies within 1e-5 of a kink are left out of the
    per-pixel comparison: there fp32 rounding in either implementation may pick the other side."""
    from dirt_b200 import matrices
    B, H, W = 64, 512, 512
    g = _gen(26)
    gbuffer = torch.rand(B, H, W, 10, generator=g, device=DEV)
    gbuffer[..., 0] = (gbuffer[..., 0] > 0.2).float()
    gbuffer[..., 1:4] = gbuffer[..., 1:4] * 2 - 1
    gbuffer[..., 7:] = torch.nn.functional.normalize(gbuffer[..., 7:] - 0.5, dim=-1)
    view = matrices.compose(matrices.translation([0., -1.5, -3.5]), matrices.rodrigues([-0.3, 0., 0.])).to(DEV)
    light = torch.nn.functional.normalize(torch.tensor([1., -0.3, -0.5], device=DEV), dim=0)
    weights = torch.rand(B, H, W, 3, generator=g, device=DEV)

    def run():
        gb, ld = gbuffer.clone().requires_grad_(True), light.clone().requires_grad_(True)
        pixels = deferred.shader_fn(gb, view, ld)
        (pixels * weights).sum().backward()
        return pixels.detach(), gb.grad, ld.grad

    px_cuda, gb_cuda, ld_cuda = run()
    px_torch, gb_torch, ld_torch = _with_restatement(monkeypatch, run)
    np.testing.assert_allclose(px_cuda.cpu().numpy(), px_torch.cpu().numpy(), rtol=2e-4, atol=2e-6)
    rel_close(px_cuda.cpu().numpy(), px_torch.cpu().numpy(), rel=2e-4, name='lighting deferred pixels')
    with torch.no_grad():   # the shader's value before its final clamp, in float64
        from dirt_b200 import lighting
        d = gbuffer.double().reshape(-1, 10)
        mask, positions, unlit, normals = d[:, :1], d[:, 1:4], d[:, 4:7], d[:, 7:]
        L64 = light.double()
        cos = normals @ -L64
        camera = torch.linalg.inv(view.double())[3, :3]
        lit = (lighting._diffuse_directional(normals, unlit, L64, torch.tensor([1., 0., 0.], device=DEV).double(), False) +
               lighting._specular_directional(positions, normals, unlit, L64, torch.ones(3, device=DEV).double(), camera,
                                              torch.tensor(6., device=DEV).double(), False) + unlit * 0.2)
        pre = lit * mask + torch.tensor([0., 0., 0.3], device=DEV).double() * (1. - mask)
        near = (cos.abs() < 1e-5) | ((pre - 1).abs() < 1e-5).any(-1) | ((pre.abs() < 1e-5) & (mask > 0)).any(-1)
        near = near.reshape(B, H, W)
    assert float(near.double().mean()) < 1e-3
    keep = ~near
    ok, ratio = rel_close(gb_cuda[keep].cpu().numpy(), gb_torch[keep].cpu().numpy(), name='lighting deferred grad_gbuffer')
    assert ok, ratio
    ok, ratio = rel_close(ld_cuda.cpu().numpy(), ld_torch.cpu().numpy(), name='lighting deferred grad_light')
    assert ok, ratio


def test_deferred_cube_through_rasterise_deferred(deferred, monkeypatch):
    """The example end to end.  The gradients of the G-buffer attributes and of the light direction are compared at
    1e-4.  The vertex gradient also has an image-space part that filters the SHADED pixels (as in the reference); the
    pixels of the two implementations differ in their last bits, and that part moved by 1.6e-3 of the largest vertex
    gradient on an H100 (the same filter run twice on identical pixels differs by atomic-order rounding only), so the
    vertex gradient is compared against 5e-3 of its largest value."""
    import dirt_b200 as dirt

    def run():
        vertices_object, vertices_clip, attributes, faces, view_matrix = deferred.scene(DEV)
        attributes.retain_grad()
        light = torch.nn.functional.normalize(torch.tensor([1., -0.3, -0.5], device=DEV), dim=0).requires_grad_(True)
        pixels = dirt.rasterise_deferred(torch.zeros([deferred.frame_height, deferred.frame_width, 10], device=DEV),
                                         vertices_clip, attributes, faces, deferred.shader_fn, [view_matrix, light])
        weights = torch.rand(pixels.shape, generator=_gen(27), device=DEV)
        (pixels * weights).sum().backward()
        return pixels.detach(), attributes.grad, light.grad, vertices_object.grad

    px_cuda, ga_cuda, gl_cuda, gv_cuda = run()
    px_torch, ga_torch, gl_torch, gv_torch = _with_restatement(monkeypatch, run)
    assert float((px_cuda != torch.tensor([0., 0., 0.3], device=DEV)).any(-1).float().mean()) > 0.1   # the cube is in view
    np.testing.assert_allclose(px_cuda.cpu().numpy(), px_torch.cpu().numpy(), rtol=2e-4, atol=2e-6)
    for name, a, b in (('attributes', ga_cuda, ga_torch), ('light', gl_cuda, gl_torch)):
        ok, ratio = rel_close(a.cpu().numpy(), b.cpu().numpy(), name='lighting deferred cube grad_' + name)
        assert ok, (name, ratio)
    worst = float((gv_cuda - gv_torch).abs().max() / gv_torch.abs().max())
    print('deferred cube: vertex gradient differs by %.2e of its largest value' % worst)
    assert worst < 5e-3, worst
