"""GPU: the GGX prefilter and its adjoint (DESIGN.md §7.12) at the map sizes it runs at, against
tests/ggx_prefilter_reference.py's rows and columns of the float64 restatement.

At S = 240 .. 2048 the kernels take the paths the dense restatement cannot reach: several compaction rounds of 256
candidate blocks (level 1 of S = 256 has 384 candidates, of S = 2048 24576), several source blocks per face with a
partial last one (S = 240, 480), and narrow lobes over many small blocks, where the cone culling decides which pairs are
summed.  A wrongly culled block weighs little against W, so membership is checked exactly: with a map that is zero but
for one texel per channel (an impulse), the texels a level is nonzero at are exactly the restatement's support, and
likewise for one-hot level gradients through the adjoint."""
import ctypes

import numpy as np
import pytest
import torch

import cubemap_ggx_restatement as ibl
import cubemap_mip_restatement as cmm
import ggx_prefilter_reference as ref
from test_gpu_cubemap import _bits_equal, _cubemap, _gen
from test_gpu_cubemap_mip import _abi, _close
from test_gpu_ibl import _prefilter, _run_abi
import variant_builds

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
TILE = 16


def _atlas(levels):
    """The whole atlas that _prefilter's level views are slices of."""
    return torch.empty(0, device=DEV).set_(levels[0].untyped_storage())


def _flat(f, r, c, Sk):
    return (np.asarray(f) * Sk + np.asarray(r)) * Sk + np.asarray(c)


def _positions(Sk, seed, n_random=8):
    """Flat texel indices of a level of Sk texels per edge where the kernels go wrong: the 8 cube corners, the 24 edge
    midpoints, both sides of a 16-block seam on every face, the first and last texel of a partial last block, and random
    texels; unique, in that order."""
    e = Sk - 1
    out = [_flat(f, r, c, Sk) for f in (0, 1) for r in (0, e) for c in (0, e)]
    out += [_flat(f, r, c, Sk) for f in range(6) for r, c in ((0, Sk // 2), (e, Sk // 2), (Sk // 2, 0), (Sk // 2, e))]
    if Sk > TILE:
        out += [_flat(f, r, c, Sk) for f in range(6) for r, c in ((TILE - 1, TILE), (TILE, TILE - 1))]
    last = (Sk - 1) // TILE * TILE
    if Sk % TILE:
        out += [_flat(f, r, c, Sk) for f in range(6) for r, c in ((last, e), (e, last), (last, last))]
    out += list(np.random.default_rng(seed).integers(0, 6 * Sk * Sk, n_random))
    return np.array(list(dict.fromkeys(int(x) for x in out)))


def _children(S, s, j):
    """The level-0 texels under texel j of box level s (its 4^s box block), flat."""
    Ss = S >> s
    f, r, c = j // (Ss * Ss), j // Ss % Ss, j % Ss
    a = np.arange(1 << s)
    rr, cc = np.meshgrid((r << s) + a, (c << s) + a, indexing='ij')
    return np.sort(_flat(f, rr, cc, S).reshape(-1))


def _parent(S, s, x):
    f, r, c = x // (S * S), x // S % S, x % S
    return _flat(f, r >> s, c >> s, S >> s)


# ---- 1. the texel and cone tables -------------------------------------------------------------------------------------


def _tables(S):
    """(texel table [n, 4], cone table [m, 4]) of S, read from the atlas at ggx_layout's offsets, as float64."""
    from dirt_b200 import _lib
    levels, _ = _prefilter(torch.zeros(1, 6, S, S, 1, device=DEV))
    atlas = _atlas(levels)
    L = ibl.level_count(S)
    pyr = sum((S >> j) ** 2 for j in range(1, L))
    weights = int(_lib.lib().dirt_cubemap_mip_atlas_bytes(1, S, 1)) // 4 + 6 * pyr
    table = (weights + 6 * pyr + 3) // 4 * 4
    n = sum(6 * (S >> k) ** 2 for k in range(L))
    m = sum(6 * (((S >> k) + TILE - 1) // TILE) ** 2 for k in range(L))
    return atlas[table:table + 4 * n].reshape(n, 4).cpu().numpy(), atlas[table + 4 * n:][:4 * m].reshape(m, 4).cpu().numpy()


@pytest.mark.parametrize('S', [240, 256, 480, 1024])
def test_texel_and_cone_tables(cuda_lib, S):
    """Directions bit for bit and solid angles within 1 ulp of the restatement's table, on every level; every texel
    corner of every 16 x 16 block, partial ones included, inside its cone."""
    table, cones = _tables(S)
    t0 = c0 = 0
    worst = 0.
    for k in range(ibl.level_count(S)):
        Sk = S >> k
        dirs, omega = ibl.texel_table(Sk)
        got = table[t0:t0 + 6 * Sk * Sk]
        t0 += 6 * Sk * Sk
        assert np.array_equal(got[:, :3].view(np.int32), dirs.reshape(-1, 3).view(np.int32)), (S, k)
        assert np.all(np.abs(got[:, 3] - omega.reshape(-1)) <= np.spacing(omega.reshape(-1))), (S, k)
        nb = (Sk + TILE - 1) // TILE
        cone = cones[c0:c0 + 6 * nb * nb].astype(np.float64).reshape(6, nb, nb, 4)
        c0 += 6 * nb * nb
        axis = cone[..., :3] / np.linalg.norm(cone[..., :3], axis=-1, keepdims=True)
        # texel corners 0 .. 16 of each block along each edge, clipped to the face (a partial block repeats its last)
        edge = np.minimum(np.arange(nb)[:, None] * TILE + np.arange(TILE + 1)[None, :], Sk)
        u = 2.0 * edge / Sk - 1.0                                     # [nb, 17]
        for f in range(6):
            cu = np.broadcast_to(u[None, :, None, :], (nb, nb, TILE + 1, TILE + 1))   # column corner of block (bi, bj)
            cv = np.broadcast_to(u[:, None, :, None], (nb, nb, TILE + 1, TILE + 1))   # row corner
            p = np.stack(ibl._face_point(f, cu, cv), -1).astype(np.float64)
            p /= np.linalg.norm(p, axis=-1, keepdims=True)
            a = axis[f][:, :, None, None, :]
            ang = np.arctan2(np.linalg.norm(np.cross(a, p), axis=-1), (a * p).sum(-1))
            excess = ang - cone[f, :, :, 3][:, :, None, None]
            worst = max(worst, float(excess.max()))
            # the fp32 acosf of a cosine near 1 leaves the half-angle up to ~1e-5 rad short (16-texel blocks of 1024^2);
            # the culling's 4e-3 rad slack covers that, and this bar keeps each cone within 1/40 of it
            assert excess.max() <= 1e-4, (S, k, f, np.unravel_index(int(excess.argmax()), excess.shape))
    print('ggx scale tables S=%d: worst corner angle beyond the cone %.3g rad' % (S, worst))


# ---- 2. forward impulses --------------------------------------------------------------------------------------------


def _source_positions(S, s, seed, n_random=8):
    return _positions(S >> s, seed + s, n_random)


@pytest.mark.parametrize('S,C,source_levels', [(240, 4, None), (256, 4, None), (480, 5, None), (1024, 4, None),
                                               (2048, 1, (1, 7))])
def test_forward_impulses(cuda_lib, S, C, source_levels):
    """One nonzero level-0 texel per channel under a chosen texel j of box level s: every output level k with
    min(k, s*) = s is nonzero exactly on column j's support, with the value w_rj v_s / W_gpu(r)."""
    L, ss = ibl.level_count(S), ibl.source_cap(S)
    checked = 0
    for s in source_levels or range(1, ss + 1):
        Ss = S >> s
        js = _source_positions(S, s, S, 8 if S < 2048 else 2)
        if S >= 2048:
            js = js[::3]
        ks = [k for k in range(1, L) if min(k, ss) == s]
        cols = {k: ref.columns(k, S, js) for k in ks}
        for g0 in range(0, len(js), C):
            group = js[g0:g0 + C]
            cube = torch.zeros(6 * S * S, C, device=DEV)
            v = torch.arange(1, C + 1, dtype=torch.float32, device=DEV)
            for ch, j in enumerate(group):
                cube[int(_children(S, s, j)[0]), ch] = v[ch]      # the box level s holds v / 4^s at j, exactly
            levels, W = _prefilter(cube.reshape(1, 6, S, S, C))
            for k in ks:
                P = levels[k - 1][0].reshape(-1, C)
                Wk = W[k - 1].reshape(-1).double().cpu().numpy()
                for ch, j in enumerate(group):
                    col = cols[k][g0 + ch]
                    got = torch.nonzero(P[:, ch]).reshape(-1).cpu().numpy()
                    assert np.array_equal(got, col.indices), (S, C, s, k, int(j), len(got), col.nnz)
                    want = col.data * (float(v[ch]) / 4 ** s) / Wk[col.indices]
                    ok, ratio = _close(P[:, ch][torch.as_tensor(col.indices, device=DEV)].double().cpu(),
                                       torch.as_tensor(want), 'ggx scale: impulse P')
                    assert ok, (S, C, s, k, int(j), ratio)
                    checked += 1
                for ch in range(len(group), C):
                    assert not P[:, ch].any()
    print('ggx scale forward impulses S=%d C=%d: %d level columns, exact membership' % (S, C, checked))


# ---- 3. adjoint impulses --------------------------------------------------------------------------------------------


def _lookups(S, C, k_texels, gout):
    """Exact-centre lookups of the given (level, flat texel) pairs at lod = level, with grad_out gout [N, C]."""
    d = np.concatenate([ref.exact_centre_directions(k, S, t) for k, t in k_texels])
    lod = np.concatenate([np.full(len(t), float(k), np.float32) for k, t in k_texels])
    assert not np.isnan(d).any()
    return torch.as_tensor(d, device=DEV), torch.as_tensor(lod, device=DEV), gout


def _ggx_atlas(lib, cube):
    """The atlas dirt_cubemap_sample_ggx builds for cube [6, S, S, C] (one lookup): all the backward pass reads."""
    S, C = cube.shape[-2], cube.shape[-1]
    atlas = torch.empty(int(lib.dirt_cubemap_ggx_atlas_bytes(1, S, C)) // 4, device=DEV)
    d, lod, out = torch.ones(1, 3, device=DEV), torch.ones(1, device=DEV), torch.empty(1, C, device=DEV)
    assert _abi(lib, 'dirt_cubemap_sample_ggx', cube, d, lod, atlas, out, 1, S, C, 1, 1) == 0
    return atlas


def _impulse_grads(lib, atlas, S, C, k, texels, det):
    """grad_cubemap [6 S^2, C] of one-hot level-k gradients: texels[i] gets grad_out 1 in channel i."""
    d, lod, gout = _lookups(S, C, [(k, texels)], torch.eye(len(texels), C, device=DEV))
    N = d.shape[0]
    nbytes = int(lib.dirt_cubemap_sample_ggx_backward_bytes(1, S, C, 1, N, det))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    gc, gd, gl = torch.empty(6 * S * S, C, device=DEV), torch.empty_like(d), torch.empty_like(lod)
    assert _abi(lib, 'dirt_cubemap_sample_ggx_backward', atlas, d, lod, gout, gc, gd, gl, 1, S, C, 1, N, det, scratch,
                ctypes.c_size_t(nbytes)) == 0
    torch.cuda.synchronize()
    return gc


def _output_positions(S, k, seed, n_random=8):
    t = _positions(S >> k, seed + k, n_random)
    return t[ref.has_exact_centre(k, S, t)]


@pytest.mark.parametrize('S,C,levels', [(240, 4, None), (256, 4, None), (480, 5, None), (1024, 4, None),
                                        (2048, 1, (1, 10))])
def test_adjoint_impulses(cuda_lib, S, C, levels):
    """A one-hot gradient at texel r of level k: grad_cubemap is nonzero exactly on row r's support expanded over the
    4^s level-0 texels of each source texel, with the value w_rj / (W_gpu(r) 4^s); the deterministic path gives the
    same bits."""
    L, ss = ibl.level_count(S), ibl.source_cap(S)
    cube = _cubemap(S, C, S)
    W = [w.reshape(-1).double().cpu().numpy() for w in _prefilter(cube[None].contiguous())[1]]
    atlas = _ggx_atlas(cuda_lib, cube)
    checked = 0
    for k in levels or range(1, L):
        s = min(k, ss)
        Ss, B = S >> s, 1 << s
        rs = _output_positions(S, k, S, 8 if S < 2048 else 2)
        if S >= 2048:
            rs = rs[::4]
        w, _ = ref.rows(k, S, rs)
        for g0 in range(0, len(rs), C):
            group = rs[g0:g0 + C]
            gc = _impulse_grads(cuda_lib, atlas, S, C, k, group, 0)
            if g0 == 0:
                assert _bits_equal(gc, _impulse_grads(cuda_lib, atlas, S, C, k, group, 1)), (S, k)
            for ch, r in enumerate(group):
                row = w[g0 + ch]
                # [level-s texel, its 4^s level-0 texels]: every one of a source texel's children carries its value
                blocks = gc[:, ch].reshape(6, Ss, B, Ss, B).permute(0, 1, 3, 2, 4).reshape(6 * Ss * Ss, B * B)
                support = torch.zeros(6 * Ss * Ss, dtype=torch.bool, device=DEV)
                support[torch.as_tensor(row.indices, device=DEV)] = True
                assert torch.equal(blocks != 0, support[:, None].expand_as(blocks)), (S, C, k, int(r), row.nnz)
                assert torch.equal(blocks, blocks[:, :1].expand_as(blocks)), (S, C, k, int(r))
                want = row.data / W[k - 1][r] / 4 ** s
                ok, ratio = _close(blocks[torch.as_tensor(row.indices, device=DEV), 0].double().cpu(),
                                   torch.as_tensor(want), 'ggx scale: impulse grad')
                assert ok, (S, C, k, int(r), ratio)
                checked += 1
    print('ggx scale adjoint impulses S=%d C=%d: %d rows, exact membership' % (S, C, checked))


# ---- 4. random maps against float64 -----------------------------------------------------------------------------------


def _sampled_outputs(Sk, seed):
    """About 1000 output texels of a level: all of a small one; else whole 16 x 16 tiles at face corners (the first
    tile of face 0, the last, partial where Sk % 16, of faces 4 and 5) and random texels on all six faces."""
    if 6 * Sk * Sk <= 1024:
        return np.arange(6 * Sk * Sk)
    last = (Sk - 1) // TILE * TILE
    out = [np.random.default_rng(seed).integers(0, 6 * Sk * Sk, 300)]
    for f, r0, c0 in ((0, 0, 0), (4, last, last), (5, last, 0)):
        r, c = np.arange(r0, min(r0 + TILE, Sk)), np.arange(c0, min(c0 + TILE, Sk))
        out.append(_flat(f, r[:, None], c[None, :], Sk).reshape(-1))
    return np.unique(np.concatenate(out))


@pytest.mark.parametrize('S,C,TB', [(240, 5, 1), (256, 3, 1), (480, 4, 1), (1024, 1, 1), (256, 3, 3)])
def test_random_maps_against_float64(cuda_lib, S, C, TB):
    """P and W of a random map at about 1000 texels of every level against the float64 sums over the full, unculled
    support."""
    L = ibl.level_count(S)
    cubes = _cubemap(S, C, S + C + TB, batch=TB)
    levels, W = _prefilter(cubes)
    box = [cmm.pyramid(cubes[b].double().cpu()) for b in range(TB)]
    worst = {}
    for k in range(1, L):
        s = ref.level_source(k, S)[0]
        idx = _sampled_outputs(S >> k, S + k)
        w, Wref = ref.rows(k, S, idx)
        ok, ratio = _close(W[k - 1].reshape(-1)[torch.as_tensor(idx, device=DEV)].double().cpu(), torch.as_tensor(Wref),
                           'ggx scale: W')
        assert ok, (S, C, k, ratio)
        worst['W'] = max(worst.get('W', 0.), ratio)
        for b in range(TB):
            want = (w @ box[b][s].reshape(-1, C).numpy()) / Wref[:, None]
            got = levels[k - 1][b].reshape(-1, C)[torch.as_tensor(idx, device=DEV)].double().cpu()
            ok, ratio = _close(got, torch.as_tensor(want), 'ggx scale: P')
            assert ok, (S, C, TB, b, k, ratio)
            worst['P'] = max(worst.get('P', 0.), ratio)
    print('ggx scale random map S=%d C=%d TB=%d: worst ratio to the bar %s' % (S, C, TB, worst))


# ---- 5. dense adjoint -----------------------------------------------------------------------------------------------


def _dense_lookups(S, C, seed):
    """One exact-centre lookup on every texel of every level k >= 1 that has one, at lod = k, random grad_out; and the
    level gradients g_k [6 S_k^2, C] float64 they make (each texel's grad_out, 0 where no lookup)."""
    L = ibl.level_count(S)
    k_texels = []
    for k in range(1, L):
        t = np.arange(6 * (S >> k) ** 2)
        k_texels.append((k, t[ref.has_exact_centre(k, S, t)]))
    n = sum(len(t) for _, t in k_texels)
    gout = torch.randn(n, C, generator=_gen(seed), device=DEV)
    d, lod, _ = _lookups(S, C, k_texels, gout)
    g, g_cpu, i = {}, gout.double().cpu().numpy(), 0
    for k, t in k_texels:
        g[k] = np.zeros((6 * (S >> k) ** 2, C))
        g[k][t] = g_cpu[i:i + len(t)]
        i += len(t)
    return d, lod, gout, g


def _sampled_texels(S, seed):
    """Level-0 texels under the seams, corners and partial edges of every box level, and random ones."""
    ss = ibl.source_cap(S)
    out = [_positions(S, seed, 40)]
    for s in range(1, ss + 1):
        j = _positions(S >> s, seed + s, 0)
        out.append(np.array([_children(S, s, x)[-1] for x in j]))
    return np.unique(np.concatenate(out))


@pytest.mark.parametrize('S,C', [(240, 5), (256, 3), (480, 4), (1024, 1)])
def test_dense_adjoint(cuda_lib, S, C):
    """Lookups on every texel of every prefiltered level: grad_cubemap at sampled texels against the float64 adjoint,
    and <out, grad_out> = <cubemap, grad_cubemap> over the whole map."""
    L, ss = ibl.level_count(S), ibl.source_cap(S)
    cube = _cubemap(S, C, 2 * S + C)
    W = {k: w.reshape(-1).double().cpu().numpy() for k, w in enumerate(_prefilter(cube[None].contiguous())[1], 1)}
    d, lod, gout, g = _dense_lookups(S, C, S + C)
    out, gc, _, _ = _run_abi(cuda_lib, cube, d, lod, gout, 0)
    lhs = (out.double() * gout.double()).sum().item()
    rhs = (cube.double() * gc.double()).sum().item()
    scale = max((out.double() * gout.double()).abs().sum().item(), (cube.double() * gc.double()).abs().sum().item())
    print('ggx scale dense adjoint S=%d C=%d: |<out, g> - <map, grad>| / sum|terms| = %.3g' % (S, C, abs(lhs - rhs) / scale))
    assert abs(lhs - rhs) <= 1e-5 * scale, (S, C, lhs, rhs, scale)
    x = _sampled_texels(S, S)
    want = sum(ref.adjoint_rows(S, s, _parent(S, s, x), g, W) / 4 ** s for s in range(1, ss + 1))
    ok, ratio = _close(gc.reshape(-1, C)[torch.as_tensor(x, device=DEV)].double().cpu(), torch.as_tensor(want),
                       'ggx scale: dense grad')
    assert ok, (S, C, ratio)
    print('ggx scale dense adjoint S=%d C=%d: %d texels, worst ratio %.3f' % (S, C, len(x), ratio))


# ---- 6. the register-staged build -----------------------------------------------------------------------------------


@pytest.mark.parametrize('S,C', [(256, 4), (480, 5)])
def test_register_staging_build_gives_the_same_bits(cuda_lib, tmp_path_factory, S, C):
    """-DDIRT_IBL_CP_ASYNC=0 stages each block through registers instead of cp.async, summing in the same order: levels,
    W, and impulse and dense-adjoint grad_cubemap are bit-identical to the product build."""
    from dirt_b200 import _lib
    staged = variant_builds._variant(tmp_path_factory, 'ibl_register_staging', {'DIRT_IBL_CP_ASYNC': 0})
    cube = _cubemap(S, C, 3 * S + C)
    want = _prefilter(cube[None].contiguous())
    saved = _lib._lib
    _lib._lib = staged
    try:
        got = _prefilter(cube[None].contiguous())
    finally:
        _lib._lib = saved
    for a, b in zip(got[0] + got[1], want[0] + want[1]):
        assert _bits_equal(a, b), S
    atlas, staged_atlas = _ggx_atlas(cuda_lib, cube), _ggx_atlas(staged, cube)
    for k in (1, 2, ibl.level_count(S) - 1):
        group = _output_positions(S, k, S)[:C]
        assert _bits_equal(_impulse_grads(staged, staged_atlas, S, C, k, group, 0),
                           _impulse_grads(cuda_lib, atlas, S, C, k, group, 0)), (S, k)
    d, lod, gout, _ = _dense_lookups(S, C, S)
    assert all(_bits_equal(a, b) for a, b in zip(_run_abi(staged, cube, d, lod, gout, 0),
                                                   _run_abi(cuda_lib, cube, d, lod, gout, 0)))


# ---- 7. SH projection at scale ----------------------------------------------------------------------------------------


@pytest.mark.parametrize('S', [480, 1024])
def test_sh_projection_at_scale(cuda_lib, S):
    """6 S^2 texels in 4096-texel chunks, the last partial at S = 480: projection and gradient against float64 torch
    on the GPU, and bit-reproducible."""
    from dirt_b200 import lighting
    C = 3
    cube = _cubemap(S, C, 4 * S)
    c = cube.clone().requires_grad_(True)
    got = lighting.cubemap_spherical_harmonics(c)
    g = torch.randn(9, C, generator=_gen(S), device=DEV)
    (got * g).sum().backward()
    ref_c = cube.double().requires_grad_(True)
    want = ibl.sh_project(ref_c)
    (want * g.double()).sum().backward()
    ok, ratio = _close(got.detach().double(), want.detach(), 'ggx scale: sh projection')
    assert ok, (S, ratio)
    ok, ratio = _close(c.grad.double(), ref_c.grad, 'ggx scale: sh grad_cubemap')
    assert ok, (S, ratio)
    assert _bits_equal(lighting.cubemap_spherical_harmonics(cube), got.detach())
