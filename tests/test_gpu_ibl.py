"""GPU: split-sum GGX image-based lighting (DESIGN.md §7.12) against tests/cubemap_ggx_restatement.py.

The prefiltered levels and their normalisers are compared with the float64 restatement at conftest.rel_close's bar; the
lookup on them bit for bit with cubemap_mip_restatement's level blend of the GPU's own levels; the gradients with float64
autograd of the restatement, evaluated at each level's float32 lookup as tests/test_gpu_cubemap_mip.py does."""
import ctypes

import numpy as np
import pytest
import torch

import cubemap_ggx_restatement as ibl
from test_gpu_cubemap import _bits_equal, _cubemap, _directions, _gen
from test_gpu_cubemap_mip import _abi, _close, _coords_of, _off_boundaries
import variant_builds

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)


def _prefilter(cubes):
    """[TB, 6, S, S, C] fp32 CUDA -> (levels 1 .. L-1 [TB, 6, S_k, S_k, C], W of levels 1 .. L-1 [6, S_k, S_k]) by
    dirt_cubemap_ggx_prefilter, read from the atlas at the offsets its header documents."""
    from dirt_b200 import _lib
    L_ = _lib.lib()
    TB, _, S, _, C = cubes.shape
    atlas = torch.empty(int(L_.dirt_cubemap_ggx_atlas_bytes(TB, S, C)) // 4, device=DEV)
    with torch.cuda.device(DEV):
        rc = L_.dirt_cubemap_ggx_prefilter(ctypes.c_void_p(cubes.data_ptr()), ctypes.c_void_p(atlas.data_ptr()), TB, S,
                                           C, ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    _lib.check(rc, 'prefilter')
    assert L_.dirt_last_launch_count() > 0
    torch.cuda.synchronize()
    lv = ibl.level_count(S)
    off = int(L_.dirt_cubemap_mip_atlas_bytes(TB, S, C)) // 4
    pyr = [sum((S >> j) ** 2 for j in range(1, k)) for k in range(lv + 1)]
    w0 = off + 6 * TB * pyr[lv] * C
    levels = [atlas[off + 6 * TB * pyr[k] * C:][:6 * TB * (S >> k) ** 2 * C].reshape(TB, 6, S >> k, S >> k, C)
              for k in range(1, lv)]
    W = [atlas[w0 + 6 * pyr[k]:][:6 * (S >> k) ** 2].reshape(6, S >> k, S >> k) for k in range(1, lv)]
    return levels, W


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize('S', [2, 4, 6, 16, 32, 64])
def test_prefilter_matches_the_restatement(cuda_lib, S, C):
    for batch in (None, 2):
        cubes = _cubemap(S, C, S + C, batch=batch)
        cubes = cubes if batch else cubes[None]
        levels, W = _prefilter(cubes.contiguous())
        for k, (got_w, want_w) in enumerate(zip(W, ibl.normalisers(S)), 1):
            ok, ratio = _close(got_w.double(), torch.as_tensor(want_w), 'ggx normalisers')
            assert ok, (S, C, k, ratio)
        for b in range(cubes.shape[0]):
            want = ibl.prefiltered_levels(cubes[b].double().cpu())
            for k, got in enumerate(levels, 1):
                ok, ratio = _close(got[b].double(), want[k], 'ggx prefilter')
                assert ok, (S, C, batch, b, k, ratio)


def _roughness(n, seed):
    """Uniform in [-0.2, 1.2], with 0, 1 and levels' own roughness among them."""
    g = _gen(seed)
    r = torch.rand(n, generator=g, device=DEV) * 1.4 - 0.2
    r[:8] = torch.tensor([0., -0., 1., 0.5, 0.25, 0.75, -1., 2.], device=DEV)
    return r


@pytest.mark.parametrize('C', [1, 3, 4, 5])
def test_lookup_is_the_level_blend_of_the_prefiltered_levels(cuda_lib, C):
    import dirt_b200 as dirt
    for k, S in enumerate([2, 6, 16, 64]):
        lv = ibl.level_count(S)
        cube = _cubemap(S, C, 70 + k)
        d = _directions(5000, 71 + k, S)
        r = _roughness(d.shape[0], 72 + k)
        levels, _ = _prefilter(cube[None].contiguous())
        want = ibl.blend_levels([cube] + [P[0] for P in levels], d, r * float(lv - 1))
        assert _bits_equal(dirt.sample_cubemap(cube, d, 'ggx', roughness=r), want), (S, C)
        for rough in (0., -0.5):
            assert _bits_equal(dirt.sample_cubemap(cube, d, 'ggx', roughness=rough),
                               dirt.sample_cubemap(cube, d, 'bilinear')), (S, C, rough)
        cubes = _cubemap(S, C, 80 + k, batch=2)
        d = torch.stack([_directions(1000, 81 + k + b, S) for b in range(2)])
        r = _roughness(2 * d.shape[1], 83 + k).reshape(2, -1)
        levels, _ = _prefilter(cubes.contiguous())
        want = torch.stack([ibl.blend_levels([cubes[b]] + [P[b] for P in levels], d[b], r[b] * float(lv - 1))
                            for b in range(2)])
        assert _bits_equal(dirt.sample_cubemap(cubes, d, 'ggx', roughness=r), want), (S, C, 'items')


def _reference_grads(cube, d, r, grad_out):
    c = cube.detach().double().cpu().requires_grad_(True)
    x = d.detach().double().cpu().requires_grad_(True)
    ro = r.detach().double().cpu().requires_grad_(True)
    x32 = d.detach().float().cpu()

    def run(c, x, ro, x32):
        if c.dim() == 5:
            return torch.stack([run(c[b], x[b], ro[b], x32[b]) for b in range(c.shape[0])])
        return ibl.sample(c, x, ro, _coords_of(x32))

    # grad_roughness is (L-1) sum_c grad_out_c (b_{m+1} - b_m): a difference of two neighbouring levels, which
    # cancels where they are close, so it is taken on the GPU's own (fp32) levels, which
    # test_prefilter_matches_the_restatement checks against the float64 ones
    cubes = cube if cube.dim() == 5 else cube[None]
    gpu_levels = _prefilter(cubes.contiguous())[0]
    ro2 = r.detach().double().cpu().requires_grad_(True)

    def run_levels(b, x, ro, x32):
        lv = [cubes[b].double().cpu()] + [P[b].double().cpu() for P in gpu_levels]
        return ibl.blend_levels(lv, x, ro * float(len(lv) - 1), _coords_of(x32))

    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        (run(c, x, ro, x32) * grad_out.double().cpu()).sum().backward()
        xd = d.detach().double().cpu()
        out = (torch.stack([run_levels(b, xd[b], ro2[b], x32[b]) for b in range(cube.shape[0])]) if cube.dim() == 5
               else run_levels(0, xd, ro2, x32))
        (out * grad_out.double().cpu()).sum().backward()
    finally:
        torch.use_deterministic_algorithms(before)
    return c.grad, (x.grad if x.grad is not None else torch.zeros_like(x)), ro2.grad


def _check_grads(cube, d, r, seed, tag, label='ggx'):
    import dirt_b200 as dirt
    grad_out = torch.randn(d.shape[:-1] + (cube.shape[-1],), generator=_gen(seed), device=DEV)
    same = _off_boundaries(d, cube.shape[-2])
    assert float(same.float().mean()) > 0.9, tag
    grad_out = grad_out * same[..., None]
    c = cube.detach().clone().requires_grad_(True)
    x = d.detach().clone().requires_grad_(True)
    ro = r.detach().clone().requires_grad_(True)
    (dirt.sample_cubemap(c, x, 'ggx', roughness=ro) * grad_out).sum().backward()
    ref = _reference_grads(cube, d, r, grad_out)
    worst = {}
    for name, got, want in zip(('grad_cubemap', 'grad_directions', 'grad_roughness'), (c.grad, x.grad, ro.grad), ref):
        ok, ratio = _close(got.cpu(), want, label + ' ' + name)
        assert ok, (tag, name, ratio)
        worst[name] = ratio
    print(tag, worst)
    return c.grad, x.grad, ro.grad


@pytest.mark.parametrize('C', [1, 3, 5])
def test_backward_matches_autograd_of_the_restatement(cuda_lib, C):
    for k, S in enumerate([2, 8, 32]):
        d = _directions(3000, 90 + k, S)
        _check_grads(_cubemap(S, C, 91 + k), d, _roughness(d.shape[0], 92 + k), 93 + k, (S, C))
    d = torch.stack([_directions(1500, 95 + b, 16) for b in range(2)])
    _check_grads(_cubemap(16, C, 97, batch=2), d, _roughness(2 * d.shape[1], 98).reshape(2, -1), 99, (16, C, 'per item'))


def _grads(cube, d, r, g):
    import dirt_b200 as dirt
    c, x, ro = (t.detach().clone().requires_grad_(True) for t in (cube, d, r))
    (dirt.sample_cubemap(c, x, 'ggx', roughness=ro) * g).sum().backward()
    return c.grad, x.grad, ro.grad


@pytest.mark.parametrize('C', [1, 3, 4])
def test_deterministic_gradient(cuda_lib, C):
    S = 32
    cube, d = _cubemap(S, C, 110), _directions(20000, 111, S)
    r = _roughness(d.shape[0], 112)
    g = torch.randn(d.shape[0], C, generator=_gen(113), device=DEV)
    default = _grads(cube, d, r, g)
    torch.use_deterministic_algorithms(True)
    try:
        first = _grads(cube, d, r, g)
        second = _grads(cube, d, r, g)
        dc = _directions(3000, 114, S)
        _check_grads(cube, dc, _roughness(dc.shape[0], 115), 116, (S, C, 'det'), label='ggx det')
    finally:
        torch.use_deterministic_algorithms(False)
    assert _bits_equal(first[0], second[0])
    assert _bits_equal(first[1], default[1]) and _bits_equal(first[2], default[2])
    assert torch.allclose(first[0], default[0], rtol=1e-4, atol=1e-5)


def test_brdf_table_matches_the_restatement(cuda_lib):
    from dirt_b200 import lighting
    table = lighting._ggx_brdf_table(DEV).cpu().numpy()
    N = ibl.BRDF_N
    assert table.shape == (N, N, 2)
    rng = np.random.default_rng(0)
    nodes = [(0, 0), (N - 1, N - 1), (0, N - 1), (N - 1, 0)] + [tuple(x) for x in rng.integers(0, N, (40, 2))]
    worst = 0.
    for i, j in nodes:
        A, B = ibl.brdf_node((i + 0.5) / N, (j + 0.5) / N)
        worst = max(worst, abs(table[i, j, 0] - A), abs(table[i, j, 1] - B))
    print('worst |GPU table - restatement|: %.3g' % worst)
    assert worst < 1e-3
    # the lookup: at nodes it is the table, and it is clamped to the outer nodes
    nv = torch.tensor([0.5 / N, 0., 1., 63.5 / N], device=DEV)
    ro = torch.tensor([0.5 / N, 0., 1., 100.5 / N], device=DEV)
    got = lighting.ggx_environment_brdf(nv, ro).cpu().numpy()
    want = table[[0, 0, N - 1, 63], [0, 0, N - 1, 100]]
    assert np.abs(got - want).max() < 1e-6


def test_furnace(cuda_lib):
    """A constant environment E: SH diffuse of its projection plus environment specular is E albedo + E (F0 A + B)."""
    from dirt_b200 import lighting
    E = torch.tensor([0.8, 1.3, 2.0], device=DEV)
    cube = E.expand(6, 16, 16, 3).contiguous()
    g = _gen(120)
    V = 500
    n = torch.randn(V, 3, generator=g, device=DEV)
    n = n / n.norm(dim=-1, keepdim=True)
    p = torch.randn(V, 3, generator=g, device=DEV) * 0.1
    cam = torch.tensor([0., 0., 4.], device=DEV)
    rough = torch.rand(V, 1, generator=g, device=DEV)
    f0 = torch.rand(V, 3, generator=g, device=DEV) * 0.2
    spec = lighting.specular_ggx_environment(p, n, rough, f0, cube, cam)
    v = cam - p
    v = v / v.norm(dim=-1, keepdim=True)
    nv = (n * v).sum(-1).abs()
    ab = lighting.ggx_environment_brdf(nv, rough[:, 0])
    want = E * (f0 * ab[:, :1] + ab[:, 1:])
    assert torch.allclose(spec, want, rtol=1e-5, atol=1e-6)
    # diffuse from the same map's SH projection: a constant map projects to L_00 = E sqrt(4 pi), the rest 0
    coeffs = lighting.cubemap_spherical_harmonics(cube)
    assert torch.allclose(coeffs[0], E * (4 * np.pi) ** 0.5, rtol=1e-5) and coeffs[1:].abs().max() < 1e-5
    albedo = torch.rand(V, 3, generator=g, device=DEV)
    diffuse = lighting.diffuse_spherical_harmonics(n, albedo, coeffs)
    assert torch.allclose(diffuse + spec, E * albedo + want, rtol=1e-4, atol=1e-5)


def test_environment_specular_gradients_reach_every_input(cuda_lib):
    from dirt_b200 import lighting
    g = _gen(130)
    V = 300
    n = torch.randn(2, V, 3, generator=g, device=DEV).requires_grad_(True)
    p = (torch.randn(2, V, 3, generator=g, device=DEV) * 0.1).requires_grad_(True)
    rough = (torch.rand(2, V, 1, generator=g, device=DEV) * 0.8 + 0.1).requires_grad_(True)
    f0 = (torch.rand(2, V, 3, generator=g, device=DEV) * 0.2).requires_grad_(True)
    cube = _cubemap(16, 3, 131, batch=2).requires_grad_(True)
    out = lighting.specular_ggx_environment(p, n, rough, f0, cube, torch.tensor([0., 0., 4.], device=DEV))
    assert out.shape == (2, V, 3) and torch.isfinite(out).all()
    out.sum().backward()
    for t in (n, p, rough, f0, cube):
        assert torch.isfinite(t.grad).all() and t.grad.abs().sum() > 0


def _run_abi(L, cube, d, lod, gout, det):
    """out, grad_cubemap, grad_directions, grad_lod of one library build through the C ABI (shared map)."""
    S, C, N = cube.shape[-2], cube.shape[-1], d.shape[0]
    atlas = torch.empty(int(L.dirt_cubemap_ggx_atlas_bytes(1, S, C)) // 4, device=DEV)
    out = torch.empty(N, C, device=DEV)
    assert _abi(L, 'dirt_cubemap_sample_ggx', cube, d, lod, atlas, out, 1, S, C, 1, N) == 0
    nbytes = int(L.dirt_cubemap_sample_ggx_backward_bytes(1, S, C, 1, N, det))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    gc, gd, gl = torch.empty_like(cube), torch.empty_like(d), torch.empty_like(lod)
    assert _abi(L, 'dirt_cubemap_sample_ggx_backward', atlas, d, lod, gout, gc, gd, gl, 1, S, C, 1, N, det, scratch,
                ctypes.c_size_t(nbytes)) == 0
    torch.cuda.synchronize()
    return out, gc, gd, gl


def test_small_grid_variant(cuda_lib, tmp_path_factory):
    """The small-grid build (grid-stride loops of many rounds): the same forward bits and deterministic gradient."""
    small = variant_builds.small_grid_library(tmp_path_factory)
    S, C = 32, 3
    cube, d = _cubemap(S, C, 140), _directions(7000, 141, S)
    lod = _roughness(d.shape[0], 142) * float(ibl.level_count(S) - 1)
    gout = torch.randn(d.shape[0], C, generator=_gen(143), device=DEV)
    a, b = _run_abi(cuda_lib, cube, d, lod, gout, 1), _run_abi(small, cube, d, lod, gout, 1)
    assert all(_bits_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize('C', [1, 3, 5])
def test_sh_projection_matches_the_restatement(cuda_lib, C):
    from dirt_b200 import lighting
    for k, S in enumerate([1, 3, 16, 64]):
        cubes = _cubemap(S, C, 150 + k, batch=2)
        c = cubes.detach().clone().requires_grad_(True)
        got = lighting.cubemap_spherical_harmonics(c)
        assert got.shape == (2, 9, C)
        g = torch.randn(2, 9, C, generator=_gen(160 + k), device=DEV)
        (got * g).sum().backward()
        for b in range(2):
            ref_c = cubes[b].detach().double().cpu().requires_grad_(True)
            want = ibl.sh_project(ref_c)
            (want * g[b].double().cpu()).sum().backward()
            ok, ratio = _close(got[b].detach().double().cpu(), want.detach(), 'sh projection')
            assert ok, (S, C, b, ratio)
            ok, ratio = _close(c.grad[b].double().cpu(), ref_c.grad, 'sh projection grad_cubemap')
            assert ok, (S, C, b, ratio)
        # shared map: the same as one item; and bit-reproducible
        one = lighting.cubemap_spherical_harmonics(cubes[0])
        assert _bits_equal(one, got[0].detach()) and _bits_equal(one, lighting.cubemap_spherical_harmonics(cubes[0]))


def test_small_grid_ibl_variant(cuda_lib, tmp_path_factory):
    """A build whose image-based-lighting kernels run on 3 CTAs and 2 items per grid: the texel and cone tables, the SH
    partial sums, and the prefilter's and its adjoint's item loops all take several rounds.  Per-item maps give the
    same bits as the product build."""
    from dirt_b200 import _lib, lighting
    import dirt_b200 as dirt
    small = variant_builds._variant(tmp_path_factory, 'ibl_small_grid',
                                    {'DIRT_IBL_MAX_BLOCKS': 3, 'DIRT_IBL_MAX_ITEMS': 2, 'DIRT_TEX_MAX_BLOCKS': 2,
                                     'DIRT_TEX_DET_GRID': 2})
    S, C, B = 32, 3, 5
    cubes = _cubemap(S, C, 170, batch=B)
    d = torch.stack([_directions(700, 171 + b, S) for b in range(B)])
    r = _roughness(B * d.shape[1], 176).reshape(B, -1)
    g = torch.randn(B, d.shape[1], C, generator=_gen(177), device=DEV)

    def run():
        c, x, ro = (t.detach().clone().requires_grad_(True) for t in (cubes, d, r))
        out = dirt.sample_cubemap(c, x, 'ggx', roughness=ro)
        sh = lighting.cubemap_spherical_harmonics(c)
        ((out * g).sum() + sh.sum()).backward()
        return out, sh, c.grad, x.grad, ro.grad

    torch.use_deterministic_algorithms(True)
    try:
        want = run()
        saved = _lib._lib
        _lib._lib = small
        try:
            got = run()
        finally:
            _lib._lib = saved
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(got, want):
        assert _bits_equal(a, b)


def test_example_fit(cuda_lib):
    """examples/ibl.py: the per-item roughness and F0 fit ends at least 10x closer to the truth than it starts."""
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location('ibl_example', os.path.join(root, 'examples', 'ibl.py'))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    cube = ex.env.procedural_cubemap(32, device=DEV)
    B = 2
    cubes = cube.expand(B, -1, -1, -1, -1).contiguous()
    truth_r, truth_f = torch.tensor([0.3, 0.55], device=DEV), torch.tensor([[0.9, 0.6, 0.3], [0.3, 0.3, 0.3]], device=DEV)
    start_r, start_f = torch.tensor([0.8, 0.1], device=DEV), torch.full((B, 3), 0.5, device=DEV)
    path_r, path_f = ex.fit_material(cubes, truth_r, truth_f, start_r, start_f)
    err = lambda r, f: float(torch.cat([(r - truth_r).abs(), (f - truth_f).abs().flatten()]).max())
    e0, e1 = err(path_r[0], path_f[0]), err(path_r[-1], path_f[-1])
    print('material fit: max |error| %.4g -> %.4g; roughness %s, F0 %s' % (e0, e1, path_r[-1].tolist(), path_f[-1].tolist()))
    assert e1 * 10 <= e0
    before, after = ex.fit_environment(cube, truth_r, truth_f, steps=40)
    print('16 x 16 environment fit: image loss %.4g -> %.4g' % (before, after))
