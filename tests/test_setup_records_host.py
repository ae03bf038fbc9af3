"""CPU: tests/setup_records.py itself.  Its restated workspace layout has the size the library asks for, and its checker
passes a workspace built from the oracle's records and rejects every way of spoiling one, each with a message that
names what is wrong."""
import numpy as np
import pytest

import kernel_paths as kp
import setup_records as sr
from dirt_b200 import scenes

VERTICES_PTR, FACES_PTR = 0x7f3a12345600, 0x7f3a9abcd000


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


# (B, H, W, C, V, F): C = 3 carves the padded colour-gradient rows, F = 0 and V = 0 empty blocks, frames that are not
# multiples of the 16x8 tile, a 1x1 frame and frames at the shading record's 65536-px limit
SIZES = [(1, 128, 128, 1, 4, 2), (2, 64, 48, 3, 62, 60), (3, 80, 96, 4, 162, 80), (5, 7, 13, 5, 14, 12), (1, 1, 1, 1, 7, 5),
         (2, 48, 64, 3, 4, 0), (1, 32, 32, 3, 0, 0), (64, 512, 512, 4, 2562, 5120), (1, 8, 65537, 3, 39, 13),
         (1, 65537, 8, 4, 39, 13), (65544, 8, 8, 4, 6, 2), (7, 17, 9, 3, 1, 1)]


@pytest.mark.parametrize('B,H,W,C,V,F', SIZES)
def test_layout_matches_the_library(L, B, H, W, C, V, F):
    lay = sr.layout(B, H, W, C, V, F)
    assert lay['bytes'] == L.dirt_workspace_bytes(B, H, W, C, V, F)
    assert lay['bytes_min'] == L.dirt_workspace_bytes_min(B, H, W, C, V, F)
    assert (lay['gc_pad'][1] > 0) == (C == 3 and B * V > 0)
    offs = [lay[n][0] for n in sr.BLOCKS]
    assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)


def test_workspace_tag_restatement():
    # FNV-1a of seven zero words, then of words that touch every byte
    h = 1469598103934665603
    for _ in range(56):
        h = (h * 1099511628211) % 2 ** 64
    assert sr.workspace_tag(0, 0, 0, 0, 0, 0, 0) == h
    assert sr.workspace_tag(VERTICES_PTR, FACES_PTR, 2, 64, 96, 1800, 600) != sr.workspace_tag(FACES_PTR, VERTICES_PTR, 2, 64, 96, 1800, 600)


def mixed_scene():
    """Two 48 x 64 images of every GPU kind: the behind-camera soup (hard faces), a large triangle, bad and NaN faces."""
    s = scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10, behind_camera=True)
    big = np.array([[-0.9, -0.9, 0.2, 1.0], [0.9, -0.8, 0.1, 1.0], [-0.7, 0.9, 0.0, 1.0], [np.nan, 0.0, 0.0, 1.0]], np.float32)
    V = s['vertices'].shape[1]
    s['vertices'] = np.concatenate([s['vertices'], np.broadcast_to(big, (2, 4, 4))], axis=1)
    s['vertex_colors'] = np.concatenate([s['vertex_colors'], np.full((2, 4, 3), 0.5, np.float32)], axis=1)
    extra = np.array([[V, V + 1, V + 2], [0, 0, 1], [0, 1, V + 99], [-1, 1, 2], [0, 1, V + 3]], np.int32)
    s['faces'] = np.concatenate([s['faces'], np.broadcast_to(extra, (2, 5, 3))], axis=1)
    return s


@pytest.fixture(scope='module')
def overflow(oracle):
    s = kp.bin_overflow_scene()
    H, W = s['background'].shape[1:3]
    ids = oracle.visibility(s['vertices'], s['faces'], H, W)[0]
    ws = sr.perfect_workspace(s['vertices'], s['faces'], s['vertex_colors'], H, W, 3, ids,
                              tag=sr.workspace_tag(VERTICES_PTR, FACES_PTR, 1, H, W, 1800, 600))
    return s, ids, ws


@pytest.fixture(scope='module')
def mixed(oracle):
    s = mixed_scene()
    H, W = s['background'].shape[1:3]
    ids = oracle.visibility(s['vertices'], s['faces'], H, W)[0]
    ws = sr.perfect_workspace(s['vertices'], s['faces'], s['vertex_colors'], H, W, 3, ids)
    return s, ids, ws


def _check(ws, s, ids, **kw):
    H, W, C = s['background'].shape[1:]
    return sr.check(ws, s['vertices'], s['faces'], H, W, C, vertex_colors=s['vertex_colors'], face_ids=ids, **kw)


def test_perfect_workspaces_pass(overflow, mixed):
    s, ids, ws = overflow
    stats = {}
    H, W = ids.shape[1:]
    assert _check(ws, s, ids, tag=sr.workspace_tag(VERTICES_PTR, FACES_PTR, 1, H, W, 1800, 600), stats=stats) is None
    assert stats['bins_past_cap'] > 0 and stats['rows_past_cap'] > 0 and stats['faces_spilled_to_large'] > 0
    s, ids, ws = mixed
    stats = {}
    assert _check(ws, s, ids, stats=stats) is None
    assert all(stats[k] > 0 for k in ('culled', 'small', 'hard', 'large')), stats


def _views(ws, s):
    B, H, W, C = s['background'].shape
    return sr.read_workspace(ws, B, H, W, C, s['vertices'].shape[1], s['faces'].shape[1])


def _face(s, kind, b=0):
    """The first face of image b that setup.cu gives `kind`."""
    H, W = s['background'].shape[1:3]
    k = sr.gpu_kind(sr.oracle_records(s['vertices'], s['faces'], H, W), H, W)[b]
    return int(np.nonzero(k == kind)[0][0])


def _mutations():
    """(name, scene, mutate(views, scene), words the message must contain)."""
    out = []

    def bins_tile(v):
        """(b, t) of a tile with at least two references in its bin."""
        b, t = np.argwhere(v['tile_count'] >= 2)[0]
        return int(b), int(t)

    def dup(v, s):
        b, t = bins_tile(v)
        v['bins'][b, t, 1] = v['bins'][b, t, 0]
    out.append(('duplicated reference', 'mixed', dup, ['duplicated reference']))

    def dropped(v, s):
        # a face that a full row list sent to the large list, lost there
        b = 0
        f = int(np.nonzero(v['face_in_large'][b])[0][0])
        n = int(v['large_count'][b])
        lst = v['large_list'][b]
        i = int(np.nonzero(lst[:n] == f)[0][0])
        lst[i] = lst[n - 1]
        v['large_count'][b] = n - 1
        v['face_in_large'][b, f] = 0
    out.append(('dropped reference', 'overflow', dropped, ['dropped reference']))

    def outside(v, s):
        b, t = bins_tile(v)
        H, W = s['background'].shape[1:3]
        exp = sr.expected(s['vertices'], s['faces'], None, H, W)
        keys = sr.binned_tiles(exp['kind'], exp['rec'], H, W)
        F = s['faces'].shape[1]
        T = np.prod(sr.tiles_of(H, W))
        here = set((keys[keys // F == b * T + t] % F).tolist())
        g = next(int(f) for f in np.nonzero(exp['kind'][b] == sr.KIND_SMALL)[0] if f not in here)
        v['bins'][b, t, 0] = g
    out.append(('reference outside the box', 'mixed', outside, ['does not touch the tile']))

    def count_plus(v, s):
        b, t = bins_tile(v)
        v['tile_count'][b, t] += 1
    out.append(('tile_count + 1', 'mixed', count_plus, ['tile_count expected']))

    def count_minus(v, s):
        b, t = bins_tile(v)
        v['tile_count'][b, t] -= 1
    out.append(('tile_count - 1', 'mixed', count_minus, ['tile_count expected']))

    def small_in_large(v, s):
        f = _face(s, sr.KIND_SMALL)
        n = int(v['large_count'][0])
        v['large_list'][0, n] = f
        v['large_count'][0] = n + 1
    out.append(('small face in the large list', 'mixed', small_in_large, ['large list holds face', 'small face']))

    for field in sr.ITP_PLANES:
        def flip(v, s, field=field):
            f = _face(s, sr.KIND_SMALL)
            v['itp'][field].view(np.uint32)[0, f] ^= 1
        out.append(('TriInterp.%s bit 0' % field, 'mixed', flip, ['TriInterp.%s' % field]))
    for field in ('zA', 'zB', 'zC'):
        for kind, layout in ((sr.KIND_SMALL, 'cov_small'), (sr.KIND_LARGE, 'cov_large'), (sr.KIND_HARD, 'cov_large')):
            def flip(v, s, field=field, kind=kind, layout=layout):
                f = _face(s, kind)
                v[layout][field].view(np.uint32)[0, f] ^= 1
            out.append(('TriCov.%s bit 0 (%s)' % (field, sr.KIND_NAMES[kind]), 'mixed', flip, ['TriCov.%s' % field]))
    for field in sr.XY_FIELDS:
        def flip(v, s, field=field):
            v['xy'][field].view(np.uint32)[0, _face(s, sr.KIND_HARD)] ^= 1
        out.append(('TriXY.%s bit 0' % field, 'mixed', flip, ['TriXY.%s' % field]))
    for field in ('sA', 'sB'):
        def flip(v, s, field=field):
            v['shade'][field].view(np.uint32)[0, _face(s, sr.KIND_SMALL)] ^= 1
        out.append(('TriShade.%s bit 0' % field, 'mixed', flip, ['TriShade.%s' % field]))

    # the fp32 roundings of float64 sums are held to one rounding: a flip of mantissa bit 12 is far past that
    def flip_sC(v, s):
        v['shade']['sC'].view(np.uint32)[0, _face(s, sr.KIND_SMALL)] ^= 1 << 12
    out.append(('TriShade.sC bit 12', 'mixed', flip_sC, ['TriShade.sC']))
    for c in range(3):
        for j in range(3):
            def flip(v, s, c=c, j=j):
                v['shade']['n'].view(np.uint32)[0, _face(s, sr.KIND_LARGE), c, j] ^= 1 << 12
            out.append(('TriShade.n[%d][%d] bit 12' % (c, j), 'mixed', flip, ['TriShade.n[%d][%d]' % (c, j)]))

    def shade_ref(v, s):
        v['shade']['ref'][0, _face(s, sr.KIND_SMALL)] += 1
    out.append(('TriShade.ref', 'mixed', shade_ref, ['TriShade.ref']))

    def swap_ids(v, s):
        f = _face(s, sr.KIND_SMALL)
        a = v['itp'][0, f]['v0'].copy()
        v['itp']['v0'][0, f] = v['itp']['v1'][0, f]
        v['itp']['v1'][0, f] = a
    out.append(('swapped vertex ids', 'mixed', swap_ids, ['TriInterp.v0']))

    def cref_itp(v, s):
        v['itp']['cref'][0, _face(s, sr.KIND_SMALL)] += 1
    out.append(('wrong TriInterp.cref', 'mixed', cref_itp, ['TriInterp.cref']))

    def cref_cov(v, s):
        v['cov_small']['cref'][0, _face(s, sr.KIND_SMALL)] += 1
    out.append(('wrong TriCov.cref', 'mixed', cref_cov, ['TriCov.cref']))

    def culled_kind(v, s):
        v['cov_small']['kind'][0, _face(s, sr.KIND_CULLED)] = sr.KIND_SMALL
    out.append(('culled face with kind 1', 'mixed', culled_kind, ['TriCov.kind', '(culled)']))

    def culled_record(v, s):
        v['itp']['sC'][0, _face(s, sr.KIND_CULLED)] = 0.0
    out.append(('culled face without its defined record', 'mixed', culled_record, ['TriInterp.sC']))

    def missing_flag(v, s):
        v['tile_flags'][0, int(np.nonzero(v['tile_flags'][0])[0][0])] = 0
    out.append(('missing tile flag', 'mixed', missing_flag, ['missing tile flag']))

    def extra_flag(v, s):
        v['tile_flags'][0, int(np.nonzero(v['tile_flags'][0] == 0)[0][0])] = 1
    out.append(('extra tile flag', 'overflow', extra_flag, ['extra tile flag']))

    def row_list_other_row(v, s):
        tx, ty = sr.tiles_of(*s['background'].shape[1:3])
        r = int(np.argmax(v['ovf_count'][0] > 0))
        v['ovf'][r, 0, 0] = (v['ovf'][r, 0, 0] + tx) % (tx * ty)
    out.append(('row-list entry of another row', 'overflow', row_list_other_row, ['not in the row']))

    def spill_flag(v, s):
        v['face_in_large'][0, _face(s, sr.KIND_SMALL)] = 1
    out.append(('face_in_large of a face that did not spill', 'mixed', spill_flag, ['face_in_large']))

    def tag(v, s):
        v['header']['tag'] ^= 1
    out.append(('header tag', 'overflow', tag, ['header: tag']))

    def error(v, s):
        v['header']['error'] = 1
    out.append(('header error', 'overflow', error, ['header: error']))
    return out


MUTATIONS = _mutations()


@pytest.mark.parametrize('name,scene,mutate,words', MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_checker_rejects(overflow, mixed, name, scene, mutate, words):
    s, ids, ws = overflow if scene == 'overflow' else mixed
    ws = ws.copy()
    mutate(_views(ws, s), s)
    H, W = ids.shape[1:]
    tag = sr.workspace_tag(VERTICES_PTR, FACES_PTR, 1, H, W, 1800, 600) if scene == 'overflow' else None
    msg = _check(ws, s, ids, tag=tag)
    assert msg is not None, name + ' was not rejected'
    for w in words:
        assert w in msg, '%s: message %r does not name it' % (name, msg)


def test_gpu_scenes_reach_every_kind_and_list_level(oracle):
    """The scenes of tests/test_gpu_setup_records.py hold faces of every GPU kind, tiles whose bin overflows into the
    row list, and rows whose list overflows into the large list."""
    import test_gpu_setup_records as g
    total = dict(culled=0, small=0, hard=0, large=0, tiles_past_bin=0, rows_past_list=0)
    for name, make in sorted(g.SCENES.items()):
        s = make()
        H, W = s['background'].shape[1:3]
        exp = sr.expected(s['vertices'], s['faces'], None, H, W)
        count = np.bincount(sr.binned_tiles(exp['kind'], exp['rec'], H, W) // s['faces'].shape[1],
                            minlength=s['faces'].shape[0] * np.prod(sr.tiles_of(H, W)))
        tx, ty = sr.tiles_of(H, W)
        row_excess = np.maximum(count - sr.BIN_CAP, 0).reshape(-1, ty, tx).sum(-1)
        for k, kind in sr.KIND_NAMES.items():
            total[kind] += int((exp['kind'] == k).sum())
        total['tiles_past_bin'] += int((count > sr.BIN_CAP).sum())
        total['rows_past_list'] += int((row_excess > sr.OVF_ROW_CAP).sum())
    print('faces and tiles the GPU scenes reach: %s' % total)
    assert all(v > 0 for v in total.values()), total
