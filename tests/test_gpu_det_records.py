"""GPU: the rasteriser backward pass term by term, against tests/det_records.py.

Deterministic path (dirt_rasterise_backward_deterministic), bit for bit under every combination of the three flags:
every channel group's code plane, the last group's float2 records, boxes and large-face list, every face's float64
partials [B*F][3][3 + C], grad_vertices, grad_vertex_colors and grad_background.  The scenes are the rare-path scenes of
kernel_paths.py (face-table overflow, flat-order taps across images, record-limit frames, depth ties), soups behind the
eye and past the guard band, one face whose box exceeds DET_WARP_BOX pixels (the CTA sweep), cfg3, cfg4 and cfg5 at a
reduced batch and sweep scene 98 of test_gpu_ref_live.py.

Default path (dirt_rasterise_backward_ex), per element: every entry of grad_vertices and grad_vertex_colors is within
gamma_n sum|t_i| + 32 u sum m_i of the float64 sum S of its n restated terms (det_records.bound).  It runs on the scenes
above, with and without shared geometry, on the 150 seeded sweep scenes of test_gpu_ref_live.py (each with its own
channel grouping) and on the four-slot variant build, where nearly every tile takes tile_generic.  Sweep scene 98,
whose position terms cancel too strongly for the tensor-wide 1e-4 bar, is asserted here like every other scene.

Face ids and pixels come from the library's forward pass (the face ids must equal the oracle's), the G-buffer from the
oracle's visibility (bit-identical to the library's, test_visibility_gbuffer_matches_oracle).  Each test prints its
worst |g - S| / bound per tensor."""
import ctypes

import numpy as np
import pytest

import det_records as dr
import kernel_paths as kp
import variant_builds
from test_gpu_paths import _p, _stream, abi_backward, abi_forward
from test_gpu_ref_live import SWEEP_SCENES, sweep_scene

pytestmark = pytest.mark.gpu


def _guard_band_soup():
    from dirt_b200 import scenes
    s = scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=3, seed=10, behind_camera=True)
    s['vertices'][:, ::7, 0] *= 4000.0
    return s


def _scenes():
    from dirt_b200 import scenes
    return {
        'overflow_c4_1_3_W62': lambda: (kp.overflow_scene(4, 62), [1, 3]),
        'overflow_c7_W64': lambda: (kp.overflow_scene(7, 64), None),
        'full_table_c3_W64': lambda: (kp.full_table_scene(3, 64), None),
        'flat_order_c4_1_3_W35': lambda: (kp.flat_order_scene(4, 35, seed=35), [1, 3]),
        'flat_order_c3_1_1_1_W33': lambda: (kp.flat_order_scene(3, 33, seed=33), [1, 1, 1]),
        'record_limit_8x65537_c4': lambda: (kp.edge_strip(8, 65537, 4, seed=4), None),
        'record_limit_65536x8_c1': lambda: (kp.edge_strip(65536, 8, 1, seed=1), None),
        'ties_b2': lambda: (kp.coplanar_tie_scene(batch=2), None),
        'soup_behind_eye_c5': lambda: (scenes.random_soup(batch=2, width=64, height=48, n_faces=40, channels=5, seed=10,
                                                          behind_camera=True), [1, 3, 1]),
        'soup_guard_band': lambda: (_guard_band_soup(), None),
        'big_face_cta_sweep': lambda: (kp.big_triangle(96, 128, [0.5, 2.0, 1.0], 3, seed=2), None),
        'cfg3_b2': lambda: (scenes.config3(batch=2), None),
        'cfg4_b2': lambda: (scenes.config4(batch=2), None),
        'cfg5_b1': lambda: (scenes.config5(batch=1), None),
        'sweep_98': lambda: sweep_scene(98),
    }


SCENE_NAMES = list(_scenes())
_CACHE = {}


def _np(t):
    return t.cpu().numpy()


def _prepared(L, oracle, s, groups, seed=0):
    """The library's forward pixels and face ids, seeded grad_pixels, the oracle's G-buffer and the restatement (no
    flags), with the CUDA tensors of the call."""
    import torch
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.items()}
    B, H, W, C = s['background'].shape
    pixels = torch.empty_like(t['background'])
    ids = torch.empty((B, H, W), dtype=torch.int32, device='cuda')
    abi_forward(L, t['background'], t['vertices'], t['vertex_colors'], t['faces'], pixels, ids)
    ids_o, gbuf = oracle.visibility(s['vertices'], s['faces'], H, W)
    ids_np, px_np = _np(ids), _np(pixels)
    assert np.array_equal(ids_np, ids_o), 'the library\'s face ids differ from the oracle\'s'
    gp_np = np.random.default_rng(seed).standard_normal(px_np.shape).astype(np.float32)
    groups = dr.groups_of(C, groups)
    G = dr.restate(s['vertices'], s['faces'], px_np, gp_np, ids_o, gbuf, groups)
    return dict(s=s, t=t, pixels=pixels, ids=ids, ids_np=ids_np, gp=torch.from_numpy(gp_np).cuda(), gp_np=gp_np,
                groups=groups, G=G)


def _scene(L, oracle, name):
    if name not in _CACHE:
        _CACHE.clear()   # one scene's buffers at a time
        s, groups = _scenes()[name]()
        _CACHE[name] = _prepared(L, oracle, s, groups)
    return _CACHE[name]


def _with_flags(G, flags):
    """The restatement under the SKIP flags: no codes, records or position terms; no colour terms."""
    out = []
    for g in G:
        g = dict(g)
        if flags & dr.SKIP_POSITION:
            g['codes'], g['rec'] = np.zeros_like(g['codes']), np.zeros_like(g['rec'])
            g['pos_p'] = g['pos_f'] = np.zeros(0, np.int64)
            g['pos_t'], g['pos_m'] = g['pos_t'][:0], g['pos_m'][:0]
        if flags & dr.SKIP_COLOUR:
            g['col_p'] = g['col_f'] = np.zeros(0, np.int64)
            g['col_t'] = g['col_t'][:0]
        out.append(g)
    return out


def _outputs(P, flags):
    import torch
    B, H, W, C = P['s']['background'].shape
    V = P['s']['vertices'].shape[1]
    lead = () if flags & dr.SHARED_GEOMETRY else (B,)
    return (torch.empty_like(P['pixels']), torch.empty(lead + (V, 4), device='cuda'),
            torch.empty(lead + (V, C), device='cuda'))


def det_backward(L, P, flags):
    """dirt_rasterise_backward_deterministic -> (grad_background, grad_vertices, grad_vertex_colors, scratch), numpy."""
    import torch
    t, groups = P['t'], P['groups']
    B, H, W, C = P['s']['background'].shape
    V, F = P['s']['vertices'].shape[1], P['s']['faces'].shape[1]
    gb, gv, gc = _outputs(P, flags)
    n = max(int(L.dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F)), 256)
    scratch = torch.full((n,), 0xA5, dtype=torch.uint8, device='cuda')
    ws = torch.empty(int(L.dirt_workspace_bytes(B, H, W, C, V, F)), dtype=torch.uint8, device='cuda')
    garr = (ctypes.c_int * len(groups))(*groups)
    rc = L.dirt_rasterise_backward_deterministic(_p(t['vertices']), _p(t['faces']), _p(P['pixels']), _p(P['gp']),
                                                 _p(P['ids']), _p(gb), _p(gv), _p(gc), B, H, W, C, V, F, garr,
                                                 len(groups), 0, flags, _p(ws), ws.numel(), _p(scratch), n, _stream())
    assert rc == 0, L.dirt_error_string(rc)
    return _np(gb), _np(gv), _np(gc), _np(scratch)


def _first_diff(what, got, want):
    """None if got and want are equal bit for bit, else a message naming the first differing entry."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    ui = {1: np.uint8, 4: np.uint32, 8: np.uint64}[got.dtype.itemsize]
    bad = np.argwhere(got.view(ui) != want.view(ui))
    if bad.size == 0:
        return None
    i = tuple(bad[0])
    return '%s: %d entries differ, first at %s: %r, restated %r' % (what, len(bad), list(i), got[i], want[i])


def check_deterministic(L, P, flags, label):
    s = P['s']
    B, H, W, C = s['background'].shape
    V, F = s['vertices'].shape[1], s['faces'].shape[1]
    G = _with_flags(P['G'], flags)
    gb, gv, gc, scratch = det_backward(L, P, flags)
    got = dr.read_scratch(scratch, B, H, W, C, V, F)
    part = dr.face_partials(G, (B, H, W), F, C)
    dv, dc = dr.vertex_sums(part, s['faces'], V, C, shared=bool(flags & dr.SHARED_GEOMETRY))
    last = G[-1]
    large = dr.large_faces(last, (B, H, W), F)
    checks = [('code plane %d' % i, got['codes'][i], g['codes']) for i, g in enumerate(G)]
    checks += [('records (last group)', got['rec'], last['rec']),
               ('boxes (last group)', got['boxes'], dr.boxes(last, (B, H, W), F)),
               ('large faces (last group)', np.sort(got['large'][:got['large_count']]), large.astype(np.int32)),
               ('face partials', got['partial'], part),
               ('grad_vertices', gv.reshape(-1, 4), dv), ('grad_vertex_colors', gc.reshape(-1, C), dc)]
    if not flags & dr.SKIP_COLOUR:
        checks.append(('grad_background', gb, dr.grad_background(P['ids_np'], P['gp_np'])))
    for what, a, b in checks:
        msg = _first_diff(what, a, b)
        assert msg is None, '%s flags=%d: %s' % (label, flags, msg)
    return len(large)


def check_default(L, P, flags, label):
    """The default path's vertex gradients, each within its fp32 bound; -> the worst ratios."""
    s = P['s']
    B, H, W, C = s['background'].shape
    V = s['vertices'].shape[1]
    gb, gv, gc = _outputs(P, flags)
    abi_backward(L, P['t']['vertices'], P['t']['faces'], P['pixels'], P['gp'], P['ids'], gb, gv, gc, P['groups'], flags)
    sv, sc = dr.term_sums(_with_flags(P['G'], flags), s['faces'], V, C, shared=bool(flags & dr.SHARED_GEOMETRY))
    ratios = {}
    for what, got, sums in (('grad_vertices', _np(gv).reshape(-1, 4), sv), ('grad_vertex_colors', _np(gc).reshape(-1, C), sc)):
        ratio, bad = dr.bound_ratio(got, sums)
        ratios[what] = ratio
        assert bad is None, '%s flags=%d: %s[%d, %d] = %.9g, its %d restated terms sum to %.9g, bound %.3g' % (
            label, flags, what, bad[0], bad[1], got[bad], sums[3][bad], sums[0][bad], dr.bound(*sums[1:])[bad])
    print('%s flags=%d: worst |g - S| / bound: grad_vertices %.4f, grad_vertex_colors %.4f' % (
        label, flags, ratios['grad_vertices'], ratios['grad_vertex_colors']))
    return ratios


# ---- the deterministic path, bit for bit ----------------------------------------------------------------------------------

@pytest.mark.parametrize('flags', range(8))
@pytest.mark.parametrize('name', SCENE_NAMES)
def test_deterministic_bit_for_bit(cuda_lib, oracle, name, flags):
    P = _scene(cuda_lib, oracle, name)
    n_large = check_deterministic(cuda_lib, P, flags, name)
    if name == 'big_face_cta_sweep' and not flags & dr.SKIP_COLOUR:
        assert n_large == 1, 'the big face should be swept by the CTA pass'
    if flags == 0:
        G = P['G']
        seen = set(np.unique(np.concatenate([g['codes'].ravel() for g in G])).tolist())
        print('%s: codes seen %s, %d position and %d colour terms' % (
            name, sorted(seen), sum(len(g['pos_p']) for g in G), sum(len(g['col_p']) for g in G)))


# ---- the default path, per element ------------------------------------------------------------------------------------------

@pytest.mark.parametrize('flags', [0, dr.SHARED_GEOMETRY])
@pytest.mark.parametrize('name', SCENE_NAMES)
def test_default_within_fp32_bound(cuda_lib, oracle, name, flags):
    check_default(cuda_lib, _scene(cuda_lib, oracle, name), flags, name)


@pytest.mark.parametrize('seed', range(SWEEP_SCENES))
def test_default_sweep_within_fp32_bound(cuda_lib, oracle, seed):
    """The seeded sweep of test_gpu_ref_live.py, each scene with its own channel grouping; scene 98 included."""
    s, groups = sweep_scene(seed)
    B, H, W, C = s['background'].shape
    P = _prepared(cuda_lib, oracle, s, groups, seed=seed)
    check_default(cuda_lib, P, 0, 'sweep seed=%d (B=%d %dx%d C=%d groups=%s)' % (seed, B, W, H, C, groups))


@pytest.fixture(scope='session')
def four_slot_lib(cuda_lib, tmp_path_factory):
    return variant_builds.four_slot_library(tmp_path_factory)


def _four_slot_scenes():
    from dirt_b200 import scenes
    out = {}
    for channels, groups in kp.OVERFLOW_CHANNELS:
        out['overflow C=%d groups=%s' % (channels, groups)] = lambda c=channels, g=groups: (kp.overflow_scene(c, 64), g)
    for channels, groups in kp.FLAT_ORDER_CHANNELS:
        out['flat order C=%d groups=%s' % (channels, groups)] = \
            lambda c=channels, g=groups: (kp.flat_order_scene(c, 37, seed=37), g)
    for channels in (1, 3, 4, 5):
        out['soup C=%d' % channels] = lambda c=channels: (scenes.random_soup(batch=2, width=61, height=45, n_faces=70,
                                                                             channels=c, seed=c), None)
    out['sweep seed=98'] = lambda: sweep_scene(98)
    return out


@pytest.mark.parametrize('name', list(_four_slot_scenes()))
def test_four_slot_within_fp32_bound(four_slot_lib, oracle, name):
    s, groups = _four_slot_scenes()[name]()
    P = _prepared(four_slot_lib, oracle, s, groups)
    for flags in (0, dr.SHARED_GEOMETRY):
        check_default(four_slot_lib, P, flags, 'slots=4 ' + name)
