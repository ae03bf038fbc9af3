"""GPU: the kernels that cap their grid, past the cap.

(a) The small-grid variant (tests/variant_builds.py) runs every capped grid-stride loop for many rounds, the last one
partial, on modest inputs.  Whatever does not depend on the grid must come out bit-identical to the product library, with
the same dirt_last_launch_count(); the texture gradient of the default (atomic) path goes against float64 autograd
instead.  The package's calls are routed to a library by replacing dirt_b200._lib.lib, and every float buffer the package
allocates starts as NaN, so that a skipped round shows.

(b) The product at its shipped limits: the texture lookups one round past 2^24, the deterministic texture gradient past
one scan round, at four sort passes and past 65 536 chunk slots, and the lighting, GGX and SH models with items past two
rounds of gridDim.y and parameter-gradient totals past 2^20 reduction CTAs, against the restatements.

tests/test_launch_limits.py shows on the CPU that every scene here crosses the boundary it is there for."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

import launch_limits as ll
import kernel_paths as kp
import test_gpu_ggx_lighting as tg
import test_gpu_lighting as tl
import test_gpu_sh_lighting as ts
import texture_det_order as order
import texture_mip_restatement as mip
import variant_builds
from conftest import rel_close
from test_gpu_deterministic import det_call as raster_det_call
from test_gpu_gbuffer_derivatives import _render, abi_derivatives
from test_gpu_texture import DEV, _bits_equal, _gen, _indices, _reference_grads, ex  # noqa: F401
from test_gpu_texture_deterministic import det_call as tex_det_call
from test_gpu_texture_mip import _random_derivatives, _reference as mip_reference

pytestmark = pytest.mark.gpu

NAN = float('nan')
_EMPTY, _EMPTY_LIKE = torch.empty, torch.empty_like


@pytest.fixture(scope='module')
def small(cuda_lib, tmp_path_factory):
    return variant_builds.small_grid_library(tmp_path_factory)


def _poisoned(t):
    if t.is_floating_point():
        t.fill_(NAN)
    elif t.dtype == torch.uint8:
        t.fill_(255)
    return t


@contextlib.contextmanager
def _through(lib):
    """The package calls `lib`, and every float buffer it allocates starts as NaN (byte buffers as 0xff)."""
    from dirt_b200 import _lib
    with pytest.MonkeyPatch.context() as m:
        m.setattr(_lib, 'lib', lambda: lib)
        m.setattr(torch, 'empty', lambda *a, **k: _poisoned(_EMPTY(*a, **k)))
        m.setattr(torch, 'empty_like', lambda *a, **k: _poisoned(_EMPTY_LIKE(*a, **k)))
        yield


def _run(lib, op, x, want, grad_out, deterministic=False):
    """op(leaves) and the gradients of (out * grad_out).sum() to the inputs `want`, through `lib` ->
    (out, {key: grad}, (launches of the forward call, launches of the last backward call))."""
    leaves = {k: v.detach().clone().requires_grad_(k in want) for k, v in x.items()}
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        with _through(lib):
            out = op(leaves)
            torch.cuda.synchronize()
            n_fwd = lib.dirt_last_launch_count()
            (out * grad_out).sum().backward()
            torch.cuda.synchronize()
            n_bwd = lib.dirt_last_launch_count()
    finally:
        torch.use_deterministic_algorithms(before)
    return out.detach(), {k: leaves[k].grad for k in want}, (n_fwd, n_bwd)


def _both(cuda_lib, small, op, x, want, grad_out, exact, deterministic=False):
    """Runs op through the product and the variant: the outputs and the gradients `exact` bit for bit, the launch
    counts equal.  Returns the product's (out, grads)."""
    out0, g0, n0 = _run(cuda_lib, op, x, want, grad_out, deterministic)
    out1, g1, n1 = _run(small, op, x, want, grad_out, deterministic)
    assert not torch.isnan(out0).any()
    assert _bits_equal(out1, out0)
    for k in exact:
        assert not torch.isnan(g0[k]).any(), k
        assert _bits_equal(g1[k], g0[k]), k
    assert n1 == n0
    return (out0, g0), (out1, g1)


def _close(a, b, name, tag):
    ok, ratio = rel_close(a.detach().cpu().numpy(), b.detach().cpu().numpy(), name=name)
    assert ok, (tag, ratio)


# ---- (a) the small-grid variant against the product -------------------------------------------------------------------

@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', ll.VAR_TEX_CHANNELS)
def test_variant_texture_lookup(ex, cuda_lib, small, mode, C):
    import dirt_b200 as dirt
    H, W = ll.VAR_TEX_SHAPE
    tex = torch.rand(H, W, C, generator=_gen(C), device=DEV)
    idx = _indices(H, W, ll.VAR_TEX_LOOKUPS, 10 + C)
    gout = torch.rand(idx.shape[0], C, generator=_gen(20 + C), device=DEV) + 0.5
    op = lambda l: dirt.sample_texture(l['tex'], l['idx'], mode=mode)   # noqa: E731
    x = dict(tex=tex, idx=idx)
    (out, g0), (_, g1) = _both(cuda_lib, small, op, x, ['tex', 'idx'], gout, ['idx'])
    assert _bits_equal(out, ex.sample_texture(tex, idx, mode=mode))
    ref_t, ref_i = _reference_grads(ex, tex, idx, gout, mode)
    _close(g0['idx'], ref_i, 'launch limits texture grad_indices', (mode, C))
    for g in (g0, g1):   # atomics: order-dependent
        _close(g['tex'], ref_t, 'launch limits texture grad_texture', (mode, C))
    # the deterministic texture gradient: bit for bit, and the restated order
    (_, d0), (_, d1) = _both(cuda_lib, small, op, x, ['tex', 'idx'], gout, ['tex', 'idx'], deterministic=True)
    want = order.grad_texture((1, H, W, C), idx[None].cpu().numpy(), gout[None].cpu().numpy(), mode)[0]
    assert np.array_equal(d0['tex'].cpu().numpy().view(np.int32), want.view(np.int32))


@pytest.mark.parametrize('C', ll.VAR_DET_LONG_CHANNELS)
def test_variant_deterministic_texture_with_listed_texels(cuda_lib, small, C):
    """Every texel has more than DET_CHUNK terms: the chunk and finish kernels loop over slots and texels."""
    TH, TW = ll.VAR_DET_LONG
    tex = torch.rand(1, TH, TW, C, generator=_gen(30 + C), device=DEV)
    idx = torch.from_numpy(ll.det_long_indices()).to(DEV)[None].contiguous()
    gout = torch.rand(idx.shape[:-1] + (C,), generator=_gen(31 + C), device=DEV) + 0.5
    got = []
    for L in (cuda_lib, small):
        with _through(L):
            gt, gi, _ = tex_det_call(tex, idx, gout)
            torch.cuda.synchronize()
            got.append((gt, gi, L.dirt_last_launch_count()))
    assert _bits_equal(got[1][0], got[0][0]) and _bits_equal(got[1][1], got[0][1]) and got[1][2] == got[0][2]
    want = order.grad_texture(tuple(tex.shape), idx.cpu().numpy(), gout.cpu().numpy())
    assert np.array_equal(got[0][0].cpu().numpy().view(np.int32), want.view(np.int32))


def _abi_pyramid(L, tex):
    TB, TH, TW, C = tex.shape
    pyr = torch.full((L.dirt_texture_mip_pyramid_bytes(TB, TH, TW, C) // 4,), NAN, device=DEV)
    assert L.dirt_texture_mip_build(ctypes.c_void_p(tex.data_ptr()), ctypes.c_void_p(pyr.data_ptr()), TB, TH, TW, C,
                                    ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)) == 0
    torch.cuda.synchronize()
    return pyr, L.dirt_last_launch_count()


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('C', [1, 3, 5])
def test_variant_trilinear_lookup_and_pyramid(cuda_lib, small, C, deterministic):
    import dirt_b200 as dirt
    TB, TH, TW = ll.VAR_MIP_SHAPE
    tex = torch.rand(TB, TH, TW, C, generator=_gen(40 + C), device=DEV)
    p0, p1 = _abi_pyramid(cuda_lib, tex), _abi_pyramid(small, tex)
    assert _bits_equal(p1[0], p0[0]) and p1[1] == p0[1]
    assert _bits_equal(p0[0], torch.cat([t.reshape(-1) for t in mip.pyramid(tex)[1:]]))
    idx = torch.stack([_indices(TH, TW, ll.VAR_TEX_LOOKUPS, 41 + b) for b in range(TB)])
    der = _random_derivatives(idx[..., 0].numel(), mip.level_count(TH, TW), 42).reshape(idx.shape[:-1] + (4,))
    gout = torch.randn(idx.shape[:-1] + (C,), generator=_gen(43), device=DEV)
    op = lambda l: dirt.sample_texture(l['tex'], l['idx'], mode='trilinear', derivatives=der)   # noqa: E731
    exact = ['tex', 'idx'] if deterministic else ['idx']
    (out, g0), (_, g1) = _both(cuda_lib, small, op, dict(tex=tex, idx=idx), ['tex', 'idx'], gout, exact, deterministic)
    for b in range(TB):
        ref_out, ref_t, ref_i = mip_reference(tex[b], idx[b], der[b], gout[b])
        _close(out[b], ref_out, 'launch limits trilinear out', b)
        _close(g0['idx'][b], ref_i, 'launch limits trilinear grad_indices', b)
        for g in (g0, g1):
            _close(g['tex'][b], ref_t, 'launch limits trilinear grad_texture', b)


def _lighting_cases():
    from dirt_b200 import lighting
    cases = {}
    for model in ('diffuse_directional', 'diffuse_point', 'specular_directional'):
        cases[model] = (lambda seed, lead, V, C, per_item: tl._inputs(seed, lead, V, C, per_item),
                        lambda x, m=model: tl._op(lighting, m, x, True), lambda x, m=model: tl._ref(lighting, m, x, True),
                        tl.ARGS[model])
    for model, point in (('ggx', False), ('ggx_point', True)):
        cases[model] = (lambda seed, lead, V, C, per_item, p=point: tg._inputs(seed, p, lead, V, C, per_item),
                        lambda x, p=point: tg._op(lighting, p, x, False), lambda x, p=point: tg._ref(lighting, p, x, False),
                        tg.KEYS)
    cases['sh'] = (ts._inputs, lambda x: ts._op(lighting, x), lambda x: ts._ref(lighting, x), ts.KEYS)
    return cases


LIGHTING = sorted(ll.LIGHT_MODELS)


@pytest.mark.parametrize('per_item', [True, False])
@pytest.mark.parametrize('C', ll.VAR_LIGHT_CHANNELS)
@pytest.mark.parametrize('model', LIGHTING)
def test_variant_lighting(cuda_lib, small, model, C, per_item):
    """No atomics: the outputs and every gradient bit for bit."""
    make, op, _, keys = _lighting_cases()[model]
    x = make(50 + C, (ll.VAR_LIGHT_B,), ll.VAR_LIGHT_V, C, per_item)
    gout = torch.rand(op(x).shape, generator=_gen(51), device=DEV) + 0.5
    _both(cuda_lib, small, op, x, keys, gout, keys)


@pytest.mark.parametrize('mesh', ['icosphere', 'fan'])
def test_variant_normals(cuda_lib, small, mesh):
    from dirt_b200 import lighting
    v, f = ll.normals_meshes()[mesh]
    g = np.random.default_rng(60)
    n = ll.VAR_NORMALS_ITEMS
    items = v[None] * (1. + 0.1 * g.random((n, 1, 1))) + 0.1 * g.standard_normal((n, 1, 3))
    x = dict(v=torch.tensor(items, dtype=torch.float32, device=DEV))
    faces = torch.tensor(f, device=DEV)
    gout = torch.rand(x['v'].shape, generator=_gen(61), device=DEV) + 0.5
    _both(cuda_lib, small, lambda l: lighting.vertex_normals(l['v'], faces), x, ['v'], gout, ['v'])
    _both(cuda_lib, small, lambda l: lighting.vertex_normals_pre_split(l['v'], faces.long()), x, ['v'], gout, ['v'])


def test_variant_gbuffer_derivatives(cuda_lib, small):
    from dirt_b200 import scenes
    s = scenes.random_soup(**ll.VAR_DERIV_SOUP)
    t, ids, ws = _render(cuda_lib, s)
    args = (t['vertices'], t['faces'], t['vertex_colors'], ids)
    for first, count in ((0, 1), (2, 2), (1, 4), (1, 3), (0, 6)):
        want = abi_derivatives(cuda_lib, *args, first, count, ws)
        n0 = cuda_lib.dirt_last_launch_count()
        got = abi_derivatives(small, *args, first, count, ws)
        assert not torch.isnan(want).any() and _bits_equal(got, want), (first, count)
        assert small.dirt_last_launch_count() == n0


@pytest.mark.parametrize('channels', [1, 3, 4, 7])
def test_variant_deterministic_rasteriser_backward(cuda_lib, small, oracle, channels):
    from dirt_b200 import scenes
    for tag, s in (('fans', kp.overflow_scene(channels, ll.VAR_OVERFLOW_W)),
                   ('soup', scenes.random_soup(channels=channels, **ll.VAR_SOUP))):
        t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in s.items()}
        pixels_o, ids_o = oracle.forward(**s, return_face_ids=True)
        pixels, ids = torch.from_numpy(pixels_o).to(DEV), torch.from_numpy(ids_o).to(DEV)
        gp = torch.from_numpy(np.random.default_rng(channels).standard_normal(pixels_o.shape).astype(np.float32)).to(DEV)
        B, V, C = pixels.shape[0], t['vertices'].shape[1], channels
        got = []
        for L in (cuda_lib, small):
            out = (torch.full_like(pixels, NAN), torch.full((B, V, 4), NAN, device=DEV), torch.full((B, V, C), NAN, device=DEV))
            with _through(L):
                raster_det_call(t, pixels, gp, ids, out=out)
                torch.cuda.synchronize()
            got.append(out + (L.dirt_last_launch_count(),))
        for a, b in zip(got[0][:3], got[1][:3]):
            assert not torch.isnan(a).any() and _bits_equal(b, a), tag
        assert got[1][3] == got[0][3], tag


# ---- (b) the product at its shipped limits ------------------------------------------------------------------------------

SLICE = 1 << 22


def _big_indices(H, W, n, seed):
    """n lookups in [-3H, 3H) x [-3W, 3W), with the edge values of test_gpu_texture._indices at the start."""
    edge = _indices(H, W, 0, seed)
    rnd = (torch.rand(n - edge.shape[0], 2, generator=_gen(seed), device=DEV) * 6 - 3) * torch.tensor([H, W], device=DEV,
                                                                                                      dtype=torch.float32)
    return torch.cat([edge, rnd])


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', [3, 4])
def test_product_texture_lookup_past_two_to_the_24(ex, cuda_lib, mode, C):
    """2^24 + 4099 lookups, one round past the cap; a 61 x 67 texture that about 4000 lookups share per texel, under a
    positive grad_out."""
    H, W, n = 61, 67, ll.TEX_LOOKUPS
    tex = torch.rand(H, W, C, generator=_gen(70 + C), device=DEV)
    idx = _big_indices(H, W, n, 71 + C)
    gout = torch.rand(n, C, generator=_gen(72 + C), device=DEV) + 0.5
    import dirt_b200 as dirt
    out, g, _ = _run(cuda_lib, lambda l: dirt.sample_texture(l['tex'], l['idx'], mode=mode), dict(tex=tex, idx=idx),
                     ['tex', 'idx'], gout)
    ref_t = torch.zeros(tex.shape, dtype=torch.float64, device=DEV)
    for s in range(0, n, SLICE):
        sl = slice(s, s + SLICE)
        assert _bits_equal(out[sl], ex.sample_texture(tex, idx[sl], mode=mode)), s
        rt, ri = _reference_grads(ex, tex, idx[sl], gout[sl], mode)
        ref_t += rt
        _close(g['idx'][sl], ri, 'launch limits texture grad_indices', (mode, C, s))
    _close(g['tex'], ref_t, 'launch limits texture grad_texture', (mode, C))


@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
@pytest.mark.parametrize('C', ll.GENERIC_CHANNELS)
def test_product_generic_forward_past_two_to_the_24_elements(ex, cuda_lib, mode, C):
    import dirt_b200 as dirt
    H, W, n = 29, 31, ll.generic_lookups(C)
    tex = torch.rand(H, W, C, generator=_gen(80 + C), device=DEV)
    idx = _big_indices(H, W, n, 81 + C)
    with _through(cuda_lib):
        out = dirt.sample_texture(tex, idx, mode=mode)
    assert _bits_equal(out, ex.sample_texture(tex, idx, mode=mode))


@pytest.mark.parametrize('deterministic', [False, True])
def test_product_trilinear_lookup_past_two_to_the_24(cuda_lib, deterministic):
    """Lambda in [-2, 3): levels 0 .. 3 are read, the coarsest of them by about 17 000 terms per texel.  (Millions of
    lookups on the 12 texels of the top level would measure the default path's fp32 atomic sums, not its loops.)"""
    import dirt_b200 as dirt
    (H, W), C, n = ll.MIP_SMALL, 3, ll.TEX_LOOKUPS
    tex = torch.rand(H, W, C, generator=_gen(90), device=DEV)
    idx = _big_indices(H, W, n, 91)
    der = _random_derivatives(n, 1, 92)   # lambda in [-2, L + 2) for L = 1
    gout = torch.rand(n, C, generator=_gen(93), device=DEV) + 0.5
    op = lambda l: dirt.sample_texture(l['tex'], l['idx'], mode='trilinear', derivatives=der)   # noqa: E731
    out, g, _ = _run(cuda_lib, op, dict(tex=tex, idx=idx), ['tex', 'idx'], gout, deterministic)
    ref_t = torch.zeros(tex.shape, dtype=torch.float64, device=DEV)
    for s in range(0, n, SLICE):
        sl = slice(s, s + SLICE)
        ro, rt, ri = mip_reference(tex, idx[sl], der[sl], gout[sl])
        ref_t += rt
        _close(out[sl], ro, 'launch limits trilinear out', s)
        _close(g['idx'][sl], ri, 'launch limits trilinear grad_indices', s)
    _close(g['tex'], ref_t, 'launch limits trilinear grad_texture', deterministic)


def test_product_pyramid_and_its_adjoint_past_the_grid(cuda_lib):
    """A 4096 x 2048 x 9 texture: building level 1 and collapsing the level gradients onto level 0 take two rounds."""
    import dirt_b200 as dirt
    TB, TH, TW, C = ll.MIP_LARGE
    tex = torch.rand(TB, TH, TW, C, generator=_gen(100), device=DEV)
    pyr, _ = _abi_pyramid(cuda_lib, tex)
    assert _bits_equal(pyr, torch.cat([t.reshape(-1) for t in mip.pyramid(tex)[1:]]))
    del pyr
    n = ll.MIP_LARGE_LOOKUPS
    idx = _big_indices(TH, TW, n, 101)
    der = _random_derivatives(n, mip.level_count(TH, TW), 102)
    gout = torch.rand(n, C, generator=_gen(103), device=DEV) + 0.5
    op = lambda l: dirt.sample_texture(l['tex'], l['idx'], mode='trilinear', derivatives=der)   # noqa: E731
    _, g, _ = _run(cuda_lib, op, dict(tex=tex[0], idx=idx), ['tex'], gout)
    _, ref_t, _ = mip_reference(tex[0], idx, der, gout)
    _close(g['tex'], ref_t, 'launch limits trilinear grad_texture', 'large')


def _det_texture(cuda_lib, tex, idx, gout):
    with _through(cuda_lib):
        gt, gi, _ = tex_det_call(tex, idx, gout, want_indices=False)
    return gt


@pytest.mark.parametrize('case', ['scan_rounds', 'four_passes'])
def test_product_deterministic_texture_bit_for_bit(cuda_lib, case):
    """260 sort tiles (two rounds of the scan's carry); and a 4097 x 4096 texture: four sort passes, 9 rounds of the
    segment bounds and 257 of the gather."""
    (H, W), n = ll.DET_SCAN if case == 'scan_rounds' else ll.DET_PASSES
    C = 2 if case == 'scan_rounds' else 1
    tex = torch.rand(1, H, W, C, generator=_gen(110), device=DEV)
    idx = _big_indices(H, W, n, 111)[None].contiguous()
    gout = torch.randn(1, n, C, generator=_gen(112), device=DEV)
    got = _det_texture(cuda_lib, tex, idx, gout)
    want = order.grad_texture(tuple(tex.shape), idx.cpu().numpy(), gout.cpu().numpy())
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32)), case


def test_product_deterministic_texture_past_the_chunk_grid(ex, cuda_lib):
    """3 * 2^25 lookups into a 2 x 2 texture: 98 304 chunk slots, one and a half rounds of the chunk kernel's 65 536
    warps.  Against float64 autograd in slices, and bit-identical on a repeat."""
    (H, W), n = ll.DET_SLOTS
    tex = torch.rand(1, H, W, 1, generator=_gen(120), device=DEV)
    idx = (torch.rand(1, n, 2, generator=_gen(121), device=DEV) * 6 - 3)
    gout = torch.rand(1, n, 1, generator=_gen(122), device=DEV) + 0.5
    first = _det_texture(cuda_lib, tex, idx, gout)
    assert _bits_equal(_det_texture(cuda_lib, tex, idx, gout), first)
    ref_t = torch.zeros(tex.shape[1:], dtype=torch.float64, device=DEV)
    for s in range(0, n, 1 << 24):
        ref_t += _reference_grads(ex, tex[0], idx[0, s:s + (1 << 24)], gout[0, s:s + (1 << 24)], 'bilinear')[0]
    _close(first[0], ref_t, 'launch limits deterministic grad_texture', '2x2')


@pytest.mark.parametrize('per_item', [True, False])
@pytest.mark.parametrize('model', LIGHTING)
def test_product_lighting_past_the_item_grid(cuda_lib, model, per_item):
    """131 077 items of 33 points; per-item parameter gradients past 2^20 reduction CTAs.  Forward and gradients against
    float64 autograd of the restatement; the items around each round of gridDim.y bit-identical alone and in the
    batch."""
    make, op, ref, keys = _lighting_cases()[model]
    C = ll.LIGHT_MODELS[model]
    x = make(130, (ll.LIGHT_B,), ll.LIGHT_V, C, per_item)
    if 'shin' in x:
        # shininess in [2, 10): for s < 2 the factor t^(s-1) of d t^s / dt, at the highlight's rim (t ~ 1e-6, where the
        # fp32 cosine keeps a few per cent), carries that rounding past the bar, and 4.3M points of random items find
        # such rims.  That is the model's fp32 accuracy, which test_gpu_lighting.py measures, not the loops.
        x['shin'] = x['shin'] + 1.
    gout = torch.rand(op(x).shape, generator=_gen(131), device=DEV) + 0.5
    out, g, _ = _run(cuda_lib, op, x, keys, gout)
    want, g64, _ = _run(cuda_lib, lambda l: ref({k: v.double() for k, v in l.items()}), x, keys, gout.double())
    _close(out, want, 'launch limits %s fwd' % model, per_item)
    for k in keys:
        _close(g[k], g64[k], 'launch limits %s grad %s' % (model, k), (per_item, k))
    if not per_item:
        return
    for b in ll.LIGHT_ITEMS:
        alone = {k: v[b:b + 1] for k, v in x.items()}
        out_b, g_b, _ = _run(cuda_lib, op, alone, keys, gout[b:b + 1])
        assert _bits_equal(out_b[0], out[b]), b
        for k in keys:
            assert _bits_equal(g_b[k][0], g[k][b]), (b, k)
