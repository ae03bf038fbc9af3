"""CPU: tests/det_records.py, the term-by-term restatement of the rasteriser's deterministic backward pass, against the
CPU oracle.  Its dilation codes (attempt and row bit included) equal the oracle's, pixel for pixel and channel group by
channel group; the float64 sums of its fp32 terms per vertex meet the oracle's gradients (terms formed in float64) within
the per-element bound of det_records.bound; the sums in the deterministic path's own order do too; and the restated
scratch layout has the size the library asks for."""
import numpy as np
import pytest

import det_records as dr
import kernel_paths as kp
from dirt_b200 import scenes


def _sweep(seed):
    from test_gpu_ref_live import sweep_scene
    return sweep_scene(seed)


SCENES = {
    'soup_c4': lambda: (scenes.random_soup(batch=2, width=40, height=30, n_faces=30, channels=4, seed=3), None),
    'soup_behind_c5_1_3_1': lambda: (scenes.random_soup(batch=2, width=37, height=29, n_faces=50, channels=5, seed=4,
                                                        behind_camera=True), [1, 3, 1]),
    'overflow_c4_1_3': lambda: (kp.overflow_scene(4, 62), [1, 3]),
    'flat_order_c3_1_1_1': lambda: (kp.flat_order_scene(3, 35, seed=35), [1, 1, 1]),
    'ties': lambda: (kp.coplanar_tie_scene(batch=2), None),
    'big_face': lambda: (kp.big_triangle(64, 80, [0.5, 2.0, 1.0], 3, seed=2), None),
    'cfg3_small': lambda: (scenes.config3(batch=2, width=96, height=80, level=2), None),
    'sweep_98': lambda: _sweep(98),
    'sweep_7': lambda: _sweep(7),
}


def _oracle_inputs(oracle, s, seed=0):
    B, H, W, C = s['background'].shape
    pixels = oracle.forward(**s)
    gp = np.random.default_rng(seed).standard_normal(pixels.shape).astype(np.float32)
    ids, gbuf = oracle.visibility(s['vertices'], s['faces'], H, W)
    return pixels, gp, ids, gbuf


@pytest.mark.parametrize('name', list(SCENES))
def test_codes_and_term_sums_match_the_oracle(oracle, name):
    s, groups = SCENES[name]()
    B, H, W, C = s['background'].shape
    V, F = s['vertices'].shape[1], s['faces'].shape[1]
    pixels, gp, ids, gbuf = _oracle_inputs(oracle, s)
    gb_o, gv_o, gc_o, codes_o = oracle.backward(s['vertices'], s['faces'], pixels, gp, groups, return_dilation='codes')
    G = dr.restate(s['vertices'], s['faces'], pixels, gp, ids, gbuf, groups)
    assert len(G) == len(codes_o)
    for gi, (g, co) in enumerate(zip(G, codes_o)):
        bad = np.argwhere(g['codes'] != co)
        assert bad.size == 0, '%s group %d: %d codes differ, first at [b, row, col] = %s: %d, oracle %d' % (
            name, gi, len(bad), bad[0].tolist(), g['codes'][tuple(bad[0])], co[tuple(bad[0])])
    if name in ('overflow_c4_1_3', 'ties', 'soup_c4'):
        seen = set(np.unique(np.concatenate([c.ravel() for c in codes_o])).tolist())
        assert {1, 2, 3, 5, 6, 7} <= seen, '%s: the codes seen are %s' % (name, sorted(seen))
    assert np.array_equal(dr.grad_background(ids, gp), gb_o)
    sv, sc = dr.term_sums(G, s['faces'], V, C)
    for what, got, sums in (('grad_vertices', gv_o.reshape(-1, 4), sv), ('grad_vertex_colors', gc_o.reshape(-1, C), sc)):
        ratio, bad = dr.bound_ratio(got, sums)
        print('%s: oracle %s within %.3f of the bound' % (name, what, ratio))
        assert bad is None, '%s: the oracle\'s %s at %s is %.9g, the restated terms sum to %.9g (bound %.3g)' % (
            name, what, bad, got[bad], sums[0][bad], dr.bound(*sums[1:])[bad])
    # the deterministic path's order, restated, lands within the same bound
    part = dr.face_partials(G, (B, H, W), F, C)
    dv, dc = dr.vertex_sums(part, s['faces'], V, C)
    assert dr.bound_ratio(dv, sv)[1] is None and dr.bound_ratio(dc, sc)[1] is None
    assert (dv[:, 2] == 0).all()


def test_codes_without_position_terms(oracle):
    s, groups = SCENES['soup_c4']()
    pixels, gp, ids, gbuf = _oracle_inputs(oracle, s)
    for g in dr.restate(s['vertices'], s['faces'], pixels, gp, ids, gbuf, groups, flags=dr.SKIP_POSITION):
        assert not g['codes'].any() and not g['rec'].any() and len(g['pos_p']) == 0 and len(g['col_p']) > 0
    for g in dr.restate(s['vertices'], s['faces'], pixels, gp, ids, gbuf, groups, flags=dr.SKIP_COLOUR):
        assert g['codes'].any() and len(g['col_p']) == 0


def test_segment_sums_are_sequential():
    """The restated per-thread sums add in the given order, one rounding per addition: 1 + 2^-53 + 2^-53 stays 1 left
    to right and is 1 + 2^-52 right to left."""
    e = 2.0 ** -53
    vals = np.array([[1.0], [e], [e]])
    _, s = dr._segment_sums(np.zeros(3, np.int64), np.array([0, 1, 2]), vals)
    assert s[0, 0] == 1.0
    _, s = dr._segment_sums(np.zeros(3, np.int64), np.array([2, 1, 0]), vals)
    assert s[0, 0] == 1.0 + 2 * e


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


# (B, H, W, C, V, F): C = 1..8, frames that are not multiples of anything, F = 0 and V = 0, the benched sizes
SIZES = [(1, 8, 8, 1, 3, 1), (2, 17, 9, 2, 14, 12), (3, 48, 62, 3, 400, 384), (2, 30, 40, 4, 90, 30), (1, 29, 37, 5, 150, 50),
         (4, 7, 13, 6, 7, 5), (2, 16, 35, 7, 1, 1), (1, 1, 1, 8, 5, 5), (2, 48, 64, 3, 4, 0), (1, 32, 32, 3, 0, 0),
         (64, 512, 512, 4, 2562, 5120), (64, 1024, 1024, 3, 24866, 49728), (0, 16, 16, 3, 4, 2)]


@pytest.mark.parametrize('B,H,W,C,V,F', SIZES)
def test_scratch_layout_matches_the_library(L, B, H, W, C, V, F):
    lay = dr.scratch_layout(B, H, W, C, V, F)
    assert lay['bytes'] == L.dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F)
    offs = [lay[n][0] for n in dr.SCRATCH_BLOCKS]
    assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)
    if B:
        assert lay['bytes'] >= lay['unsorted'][0] + lay['unsorted'][1]


def test_scratch_reader_round_trip():
    """read_scratch finds each block where scratch_layout puts it."""
    B, H, W, C, V, F = 2, 5, 7, 4, 6, 3
    lay = dr.scratch_layout(B, H, W, C, V, F)
    buf = np.zeros(lay['bytes'], np.uint8)
    o = lay['partial'][0]
    buf[o:o + 8] = np.array([1.5]).view(np.uint8)
    o = lay['rec'][0]
    buf[o:o + 8] = np.array([2.0, -3.0], np.float32).view(np.uint8)
    buf[lay['codes'][0] + B * H * W + 1] = 7
    v = dr.read_scratch(buf, B, H, W, C, V, F)
    assert v['partial'][0, 0, 0] == 1.5 and tuple(v['rec'][0, 0, 0]) == (2.0, -3.0) and v['codes'][1, 0, 0, 1] == 7
