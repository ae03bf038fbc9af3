"""GPU: shadow-map lookups (DESIGN.md §7.15) where test_gpu_shadow.py does not go -- maps smaller than the tap
footprint, one to four radix-sort passes and several gather rounds, many points on one texel, every subset of the
gradients, rendered maps under perspective lights with receivers on the rendered surfaces, and production map sizes.

The kernels are compared with tests/shadow_reference.py, a float64 restatement that takes every fp32 decision (base
texel, fraction, depth step) exactly as the kernels take it, so continuous random depths and receivers lying on an
occluder compare at the 1e-4 bar with no tie exclusions.  The deterministic map gradient is also compared bit for bit
with its documented summation order wherever the inputs are dyadic."""
import itertools

import numpy as np
import pytest
import torch

import shadow_reference as sr
from conftest import rel_close
from dirt_b200 import lighting, matrices
from test_gpu_shadow import _case

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
NAMES = ('visibility', 'grad_positions', 'grad_light_matrix', 'grad_shadow_map')
BIAS = 0.01


@pytest.fixture(autouse=True)
def _library(cuda_lib):
    """Skips without a CUDA device; builds the library if it is stale."""
    return cuda_lib


def _random_case(B, N, per_item, SH, SW, seed, margin=0.1):
    """Mildly perspective light matrices, points spread over the map and `margin` of its size past each edge, with
    continuous random depths, and a map of random occupancy and continuous depths: fp32 arrays."""
    g = np.random.default_rng(seed)
    nm = B if per_item else 1
    M = np.tile(np.eye(4), (nm, 1, 1))
    M[:, :3, :3] += g.uniform(-0.1, 0.1, (nm, 3, 3))
    M[:, 3, :3] += g.uniform(-0.1, 0.1, (nm, 3))
    M[:, 2, 3] = g.choice([-1., 1.], nm) * g.uniform(0.02, 0.05, nm)
    Minv = np.linalg.inv(M)
    X = g.uniform(-margin, 1 + margin, (B, N)) * SW
    Yd = g.uniform(-margin, 1 + margin, (B, N)) * SH
    z, w = g.uniform(-0.6, 0.6, (B, N)), g.uniform(0.8, 1.2, (B, N))
    h = np.stack([(X / (SW / 2) - 1) * w, (1 - Yd / (SH / 2)) * w, z, w], -1)
    p = np.einsum('bnk,bkj->bnj', h, Minv if per_item else np.broadcast_to(Minv, (B, 4, 4)))
    p = p[..., :3] / p[..., 3:]
    smap = np.stack([g.uniform(size=(nm, SH, SW)) < 0.6, g.uniform(-0.6, 0.6, (nm, SH, SW))], -1)
    if not per_item:
        M, smap = M[0], smap[0]
    return [np.asarray(x, np.float32) for x in (p, M, smap)]


def _dyadic_case(B, N, per_item, SH, SW, seed, x=None, y=None):
    """Identity light matrices, points on a 2^-12 grid of clip x and y (given as clip coordinates, or drawn over the
    map and a little past it), depths on a 2^-4 grid and grad_out on a 2^-5 grid: every fp32 step of a term is exact,
    so the deterministic map gradient can be restated bit for bit."""
    g = np.random.default_rng(seed)
    if x is None:
        x = g.integers(-200, (1 << 13) + 200, (B, N)) / 4096. - 1
        y = g.integers(-200, (1 << 13) + 200, (B, N)) / 4096. - 1
    z = g.integers(-8, 8, (B, N)) / 16. + 1 / 32.
    p = np.stack([x, y, z], -1)
    nm = B if per_item else 1
    smap = np.stack([g.uniform(size=(nm, SH, SW)) < 0.6, g.integers(-8, 8, (nm, SH, SW)) / 16.], -1)
    M = np.tile(np.eye(4), (nm, 1, 1))
    if not per_item:
        M, smap = M[0], smap[0]
    gout = g.integers(-64, 64, (B, N, 1)) / 32.
    return [np.asarray(x, np.float32) for x in (p, M, smap, gout)]


def _gpu(p, M, smap, R, softness, gout, want=(True, True, True), deterministic=False):
    """visibility and the wanted gradients (None for the others) of lighting.shadow_visibility on the GPU."""
    leaves = [torch.tensor(x, device=DEV).requires_grad_(w) for x, w in zip((p, M, smap), want)]
    torch.use_deterministic_algorithms(deterministic)
    try:
        v = lighting.shadow_visibility(*leaves, R, softness, BIAS)
        (v * torch.tensor(gout, device=DEV)).sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
    return [v.detach().cpu().numpy()] + [t.grad.cpu().numpy() if w else None for t, w in zip(leaves, want)]


def _check(got, want, tag, names=NAMES, rel=1e-4, prefix='shadow edges '):
    for g, w, name in zip(got, want, names):
        if g is None:
            continue
        ok, worst = rel_close(g, w, rel=rel, name=prefix + name)
        assert ok, (tag, name, worst)


def _ref(p, M, smap, R, softness, gout, want=(True, True, True), device='cpu'):
    vis, grads = sr.reference(p, M, smap, R, softness, BIAS, gout, want, device)
    return [vis] + list(grads)


# ---- maps smaller than the tap footprint, and one large odd map -----------------------------------------------------

SHAPES = [(1, 1), (1, 7), (7, 1), (2, 2), (3, 3), (2, 5), (5, 2), (1023, 769)]
SHAPE_IDS = ['%dx%d' % s for s in SHAPES]


@pytest.mark.parametrize('shape', SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize('R', [0, 1, 2, 3])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_map_shapes(shape, R, softness, per_item):
    """Visibility and all three gradients on the default path, and the deterministic map gradient, against the
    reference: taps that clamp onto one row or column from both sides, and a 1023 x 769 map."""
    SH, SW = shape
    B, N = 3, 400
    p, M, smap = _random_case(B, N, per_item, SH, SW, seed=SH * 31 + SW + 1000 * R + 7 * per_item + int(softness > 0))
    # one sign: on the small maps each texel sums up to 20 000 terms with float atomics, which keeps the bar's
    # relative accuracy only without cancellation (the deterministic sums are float64)
    gout = np.random.default_rng(R).uniform(0.5, 1.5, (B, N, 1)).astype(np.float32)
    want = _ref(p, M, smap, R, softness, gout)
    tag = (shape, R, softness, per_item)
    _check(_gpu(p, M, smap, R, softness, gout), want, tag)
    det = _gpu(p, M, smap, R, softness, gout, (False, False, True), deterministic=True)
    _check(det[3:], want[3:], tag, ('deterministic grad_shadow_map',))


@pytest.mark.parametrize('shape', SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize('R', [0, 1, 2, 3])
@pytest.mark.parametrize('per_item', [True, False])
def test_deterministic_order_on_map_shapes(shape, R, per_item):
    """Dyadic points, identity matrices, softness 0: the deterministic map gradient is, bit for bit, each texel's
    float64 sum of the fp32 terms in the documented order, rounded once."""
    SH, SW = shape
    B, N = 2, 1500
    p, M, smap, gout = _dyadic_case(B, N, per_item, SH, SW, seed=SH * 17 + SW + 100 * R + per_item)
    got = _gpu(p, M, smap, R, 0., gout, (False, False, True), deterministic=True)[3]
    assert np.array_equal(got, sr.deterministic_map_gradient(p, M, smap, R, BIAS, gout))


# ---- sort passes and gather rounds ----------------------------------------------------------------------------------

PASS_CASES = [
    # name, B, N, per_item, SH, SW, sort passes
    ('shared 7x1', 3, 2000, False, 7, 1, 1),
    ('per-item 1x1', 3, 2000, True, 1, 1, 1),
    ('per-item 24x40', 3, 2000, True, 24, 40, 2),
    ('per-item 2x256^2', 2, 30000, True, 256, 256, 3),
    ('per-item 17x1024^2', 17, 4000, True, 1024, 1024, 4),
    ('shared 4096^2', 2, 60000, False, 4096, 4096, 4),   # 2^24 texels: eight rounds of the gather's grid
]


@pytest.mark.parametrize('case', PASS_CASES, ids=[c[0] for c in PASS_CASES])
def test_sort_passes_and_gather_rounds(case):
    """Key counts that sort in one to four radix passes (the sorted keys end in either ping-pong buffer), and a map of
    more texels than one gather grid covers: every gradient of the deterministic call against the reference, and
    bit-identical across two calls; the default path against the reference too."""
    name, B, N, per_item, SH, SW, passes = case
    assert sr.sort_passes(B, per_item, SH, SW) == passes
    R, softness = 1, 0.02
    p, M, smap = _random_case(B, N, per_item, SH, SW, seed=SH + SW + B)
    gout = np.random.default_rng(B).standard_normal((B, N, 1)).astype(np.float32)
    want = _ref(p, M, smap, R, softness, gout, device='cuda')
    det = _gpu(p, M, smap, R, softness, gout, deterministic=True)
    again = _gpu(p, M, smap, R, softness, gout, deterministic=True)
    assert all(np.array_equal(a, b) for a, b in zip(det, again)), name
    _check(det, want, name)
    _check(_gpu(p, M, smap, R, softness, gout), want, name)


# ---- contention: many points per texel ------------------------------------------------------------------------------

def _grid_points(n, lo=-1., hi=1.):
    """n^2 dyadic clip (x, y) pairs: a 2^-12 grid from lo to hi."""
    a = lo + (np.arange(n) * ((hi - lo) * 4096 // n)) / 4096. + 1 / 8192.
    y, x = np.meshgrid(a, a, indexing='ij')
    return x.reshape(1, -1), y.reshape(1, -1)


def _contention(p, M, smap, R, softness, gout, tag, order=True):
    want = _ref(p, M, smap, R, softness, gout, device='cuda')
    _check(_gpu(p, M, smap, R, softness, gout), want, tag)
    det = _gpu(p, M, smap, R, softness, gout, (False, False, True), deterministic=True)
    _check(det[3:], want[3:], tag, ('deterministic grad_shadow_map',))
    if order and softness == 0:
        assert np.array_equal(det[3], sr.deterministic_map_gradient(p, M, smap, R, BIAS, gout)), tag


@pytest.mark.parametrize('S', [4, 16])
@pytest.mark.parametrize('R', [0, 1])
@pytest.mark.parametrize('softness', [0., 0.05])
def test_many_points_on_a_small_map(S, R, softness):
    """512^2 points on a 4 x 4 or 16 x 16 map: whole warps hit one texel at every tap."""
    x, y = _grid_points(512)
    p, M, smap, gout = _dyadic_case(1, x.size, False, S, S, seed=S + R, x=x, y=y)
    gout = np.abs(gout) + np.float32(0.5)   # one sign: the fp32 atomic sums then keep their relative accuracy
    _contention(p, M, smap, R, softness, gout, ('small map', S, R, softness))


@pytest.mark.parametrize('R', [0, 2])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_every_point_on_one_texel(R, softness, per_item):
    """20 000 points per item with one base texel, varied fractions and depths: one segment of the sort holds them
    all, and one thread of the gather sums each of the (2R+2)^2 texels they reach."""
    B, N, S = 2, 20000, 8
    g = np.random.default_rng(40 + R)
    # X in [3.5, 4.5): base column 3; clip x = X / 4 - 1 on a 2^-12 grid
    x = (g.integers(0, 1024, (B, N)) / 1024. + 3.5) / (S / 2) - 1
    y = 1 - (g.integers(0, 1024, (B, N)) / 1024. + 4.5) / (S / 2)
    p, M, smap, gout = _dyadic_case(B, N, per_item, S, S, seed=41 + R, x=x, y=y)
    look = sr.lookups(*sr._flat(p, M, smap)[:2], S, S)
    assert (look['c0'] == 3).all() and (look['r0'] == 4).all()
    _contention(p, M, smap, R, softness, gout, ('one texel', R, softness, per_item))


@pytest.mark.parametrize('shape', [(16, 16), (9, 5)], ids=['16x16', '9x5'])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_pile_ups_on_corners_and_edges(shape, softness, per_item):
    """R = 3: points piled within half a texel of the map's corners and edges, where every tap clamps and the gather
    sums the most base segments per texel."""
    SH, SW = shape
    B, N = 2, 6000
    g = np.random.default_rng(SH + SW)

    def near_edges(n, size):
        # half of the points within half a texel of the low edge, half of the high one; some spread inside
        a = np.where(g.uniform(size=(B, N)) < 0.5, g.uniform(0, 0.5, (B, N)), size - g.uniform(0, 0.5, (B, N)))
        spread = g.uniform(size=(B, N)) < 0.25
        a = np.where(spread, g.uniform(0, size, (B, N)), a)
        return np.floor(a * 1024) / 1024.

    X, Yd = near_edges(N, SW), near_edges(N, SH)
    x, y = X / (SW / 2.) - 1, 1 - Yd / (SH / 2.)
    x, y = np.round(x * 4096) / 4096., np.round(y * 4096) / 4096.
    p, M, smap, gout = _dyadic_case(B, N, per_item, SH, SW, seed=SH * SW + per_item, x=x, y=y)
    _contention(p, M, smap, 3, softness, gout, ('pile-ups', shape, softness, per_item))


# ---- the autograd surface -------------------------------------------------------------------------------------------

SUBSETS = [w for w in itertools.product((False, True), repeat=3) if any(w)]


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('softness', [0., 0.05])
@pytest.mark.parametrize('per_item', [True, False])
def test_each_subset_of_the_gradients(deterministic, softness, per_item):
    """Every non-empty subset of (positions, light matrix, map): each wanted gradient against the reference; the
    position and matrix gradients, and the deterministic map gradient, bit-identical to those of the full call."""
    B, N, SH, SW, R = 3, 3000, 24, 40, 1
    p, M, smap = _random_case(B, N, per_item, SH, SW, seed=90 + 2 * per_item + int(softness > 0))
    gout = np.random.default_rng(91).standard_normal((B, N, 1)).astype(np.float32)
    want = _ref(p, M, smap, R, softness, gout)
    full = _gpu(p, M, smap, R, softness, gout, deterministic=deterministic)
    for subset in SUBSETS:
        got = _gpu(p, M, smap, R, softness, gout, subset, deterministic)
        tag = (subset, deterministic, softness, per_item)
        _check(got, want, tag)
        assert np.array_equal(got[0], full[0]), tag
        for k in (1, 2) + ((3,) if deterministic else ()):
            assert got[k] is None or np.array_equal(got[k], full[k]), (tag, NAMES[k])


@pytest.mark.parametrize('per_item', [True, False])
def test_double_backward(per_item):
    """create_graph=True differentiates through the restatement: the first and second gradients against float64."""
    B, N, R, softness = 2, 500, 1, 0.05
    p, M, smap = [np.asarray(x, np.float32) for x in _case(B, N, per_item, seed=95 + per_item, special=False)]
    # one sign: the fp32 restatement's first map gradient is summed with float atomics, as in test_map_shapes
    gout = np.random.default_rng(96).uniform(0.5, 1.5, (B, N, 1)).astype(np.float32)

    def second(device, dtype):
        leaves = [torch.tensor(x, device=device, dtype=dtype, requires_grad=True) for x in (p, M, smap)]
        fn = lighting.shadow_visibility if device == DEV else lighting._shadow_visibility
        out = fn(*leaves, R, softness, BIAS)
        first = torch.autograd.grad((out * torch.tensor(gout, device=device, dtype=dtype)).sum(), leaves,
                                    create_graph=True)
        sum(g.square().sum() for g in first).backward()
        return [g.detach().cpu().numpy() for g in first] + [t.grad.cpu().numpy() for t in leaves]

    got, want = second(DEV, torch.float32), second(torch.device('cpu'), torch.float64)
    _check(got, want, per_item, ['first ' + n for n in NAMES[1:]] + ['second ' + n for n in NAMES[1:]])


@pytest.mark.parametrize('deterministic', [False, True])
def test_cuda_graph_capture_and_replay(deterministic):
    B, N, S = 2, 50000, 64
    p, M, smap = _random_case(B, N, True, S, S, seed=97)
    leaves = [torch.tensor(x, device=DEV, requires_grad=True) for x in (p, M, smap)]
    gout = torch.randn((B, N, 1), device=DEV)

    def step():
        for t in leaves:
            t.grad = None
        out = lighting.shadow_visibility(*leaves, 1, 0.05, BIAS)
        (out * gout).sum().backward()
        return out

    torch.use_deterministic_algorithms(deterministic)
    try:
        eager = step().detach().clone()
        eager_grads = [t.grad.clone() for t in leaves]
        side = torch.cuda.Stream(DEV)
        side.wait_stream(torch.cuda.current_stream(DEV))
        with torch.cuda.stream(side):
            step()
        torch.cuda.current_stream(DEV).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = step()
        for _ in range(2):
            for t in leaves:
                t.grad.fill_(float('nan'))
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, eager)
            assert torch.equal(leaves[0].grad, eager_grads[0]) and torch.equal(leaves[1].grad, eager_grads[1])
            if deterministic:
                assert torch.equal(leaves[2].grad, eager_grads[2])
            else:   # float atomics: the order of the additions may change
                ok, worst = rel_close(leaves[2].grad.cpu().numpy(), eager_grads[2].cpu().numpy())
                assert ok, worst
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize('deterministic', [False, True])
def test_an_item_alone_and_inside_a_batch(deterministic):
    """Visibility, position and matrix gradients bit-identical for an item alone (shared matrix and map) and inside a
    per-item batch; the deterministic map gradient too."""
    B, N, SH, SW, R, softness = 5, 5000, 32, 48, 2, 0.05
    p, M, smap = _random_case(B, N, True, SH, SW, seed=98)
    gout = np.random.default_rng(99).standard_normal((B, N, 1)).astype(np.float32)
    batch = _gpu(p, M, smap, R, softness, gout, deterministic=deterministic)
    for b in (0, 3):
        alone = _gpu(p[b], M[b], smap[b], R, softness, gout[b], deterministic=deterministic)
        for k in range(4 if deterministic else 3):
            assert np.array_equal(alone[k], batch[k][b]), (b, NAMES[k])


@pytest.mark.parametrize('deterministic', [False, True])
def test_leading_dimensions(deterministic):
    """positions [2, 3, N, 3] with matrices [2, 3, 4, 4] and maps [2, 3, SH, SW, 2]."""
    N, SH, SW, R, softness = 700, 12, 20, 1, 0.05
    p, M, smap = _random_case(6, N, True, SH, SW, seed=100)
    p, M, smap = p.reshape(2, 3, N, 3), M.reshape(2, 3, 4, 4), smap.reshape(2, 3, SH, SW, 2)
    gout = np.random.default_rng(101).standard_normal((2, 3, N, 1)).astype(np.float32)
    got = _gpu(p, M, smap, R, softness, gout, deterministic=deterministic)
    assert [x.shape for x in got] == [(2, 3, N, 1), p.shape, M.shape, smap.shape]
    _check(got, _ref(p, M, smap, R, softness, gout), deterministic)


# ---- rendered maps under perspective lights -------------------------------------------------------------------------

def _look_at(eye, target):
    """The world -> view matrix [4, 4] (row vectors) of a light at `eye` looking at `target`, up +y."""
    back = eye - target
    back = back / np.linalg.norm(back)
    right = np.cross([0., 1., 0.], back)
    right = right / np.linalg.norm(right)
    up = np.cross(back, right)
    V = np.eye(4)
    V[:3, :3] = np.stack([right, up, back], 1)
    V[3, :3] = -eye @ V[:3, :3]
    return V


def _scene():
    """A floor quad at y = 0 and a box above it, one mesh: vertices [12, 3], faces [14, 3]."""
    floor = np.array([[-1.2, 0., -1.2], [1.2, 0., -1.2], [1.2, 0., 1.2], [-1.2, 0., 1.2]])
    corners = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * 0.25
    a = 0.4
    rot = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    box = corners @ rot.T + [0.1, 0.55, -0.1]
    faces = [[0, 2, 1], [0, 3, 2]]
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
    for q in quads:
        q = [4 + i for i in q]
        faces += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    return np.concatenate([floor, box]).astype(np.float32), np.array(faces, np.int32)


def _surface_points(v, f, n, g):
    """n points uniformly on the faces, by area."""
    tri = v[f].astype(np.float64)
    area = np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    which = g.choice(len(f), n, p=area / area.sum())
    a, b = g.uniform(size=(2, n))
    flip = a + b > 1
    a, b = np.where(flip, 1 - a, a), np.where(flip, 1 - b, b)
    t = tri[which]
    return t[:, 0] + a[:, None] * (t[:, 1] - t[:, 0]) + b[:, None] * (t[:, 2] - t[:, 0])


def _interior_depths(clip, f, S):
    """Per texel centre of an S x S map: the float64 clip z of the nearest face that covers the centre (NaN where
    none does), and a mask of the texels whose centre is at least 2% of a barycentric unit from every face's edges."""
    r, c = np.meshgrid(np.arange(S), np.arange(S), indexing='ij')
    xn, yn = (c + 0.5) / (S / 2.) - 1, 1 - (r + 0.5) / (S / 2.)
    best = np.full((S, S), np.inf)
    depth = np.full((S, S), np.nan)
    clear = np.ones((S, S), bool)
    for face in f:
        cv = clip[face]   # [3, 4]
        A = np.empty((S, S, 3, 3))
        A[..., 0, :] = cv[:, 0] - xn[..., None] * cv[:, 3]
        A[..., 1, :] = cv[:, 1] - yn[..., None] * cv[:, 3]
        A[..., 2, :] = 1.
        lam = np.linalg.solve(A, np.broadcast_to([0., 0., 1.], (S, S, 3))[..., None])[..., 0]
        inside = (lam > 0.02).all(-1)
        clear &= inside | (lam < -0.02).any(-1)
        z, w = lam @ cv[:, 2], lam @ cv[:, 3]
        nearer = inside & (z / w < best)
        best = np.where(nearer, z / w, best)
        depth = np.where(nearer, z, depth)
    return depth, clear


@pytest.mark.parametrize('softness', [0., 0.005])
def test_rendered_maps_under_perspective_lights(softness):
    """shadow_map of a box over a floor from two perspective lights, receivers on both surfaces at a small bias.  The
    visibility and receiver gradient against the reference on the GPU's own map; the vertex and light-matrix gradients
    (through the map and the lookup) against the reference's map gradient fed to the CPU oracle's backward pass and
    chained through clip = (p, 1) @ M; the depth channel against float64 clip z at interior texels."""
    from oracle import oracle
    S, N, R, bias = 256, 20000, 1, 0.002
    v, f = _scene()
    eyes = np.array([[1.5, 3.0, 1.0], [-1.0, 2.5, 2.0]])
    proj = matrices.perspective_projection(1., 8., 0.75, 1.).numpy().astype(np.float64)
    M = np.stack([_look_at(e, np.zeros(3)) @ proj for e in eyes]).astype(np.float32)
    B = len(M)
    g = np.random.default_rng(7)
    recv = np.stack([_surface_points(v, f, N, g) for _ in range(B)]).astype(np.float32)
    weight = g.uniform(0.5, 1.5, (B, N, 1)).astype(np.float32)

    verts = torch.tensor(v, device=DEV, requires_grad=True)
    tM = torch.tensor(M, device=DEV, requires_grad=True)
    trecv = torch.tensor(recv, device=DEV, requires_grad=True)
    smap = lighting.shadow_map(verts.expand(B, -1, -1), torch.tensor(f, device=DEV), tM, S, S)
    vis = lighting.shadow_visibility(trecv, tM, smap, R, softness, bias)
    (vis * torch.tensor(weight, device=DEV)).sum().backward()
    got_map = smap.detach().cpu().numpy()

    # receivers on the lit side of the box are in contact with their own texels' depths: some lit, some shadowed
    vis = vis.detach().cpu().numpy()
    assert 0.1 < (vis < 0.5).mean() < 0.9
    want_vis, (g_recv, g_M_lookup, g_map) = sr.reference(recv, M, got_map, R, softness, bias, weight, device='cuda')
    _check([vis, trecv.grad.cpu().numpy()], [want_vis, g_recv], softness, ('rendered visibility', 'rendered grad_positions'))

    clip32 = torch.matmul(torch.cat([verts, torch.ones_like(verts[:, :1])], -1), tM).detach().cpu().numpy()
    _, gv, gc = oracle.backward(clip32, np.broadcast_to(f, (B,) + f.shape), got_map, g_map.astype(np.float32))
    gclip = gv.astype(np.float64)
    gclip[..., 2] += gc[..., 1]   # the depth channel's colour is clip z
    v64 = torch.tensor(v, dtype=torch.float64, requires_grad=True)
    M64 = torch.tensor(M, dtype=torch.float64, requires_grad=True)
    torch.matmul(torch.cat([v64, torch.ones_like(v64[:, :1])], -1), M64).backward(torch.tensor(gclip))
    # through the rasteriser's fp32 backward pass and the map gradient's float atomics, as test_gpu_shadow.py's pipeline
    _check([verts.grad.cpu().numpy(), tM.grad.cpu().numpy()],
           [v64.grad.numpy(), M64.grad.numpy() + g_M_lookup], softness,
           ('rendered occluder gradient', 'rendered light-matrix gradient'), rel=1e-3)

    for b in range(B):
        clip = np.concatenate([v.astype(np.float64), np.ones((len(v), 1))], 1) @ M[b].astype(np.float64)
        depth, interior = _interior_depths(clip, f, S)
        covered = interior & np.isfinite(depth)
        assert covered.sum() > S * S // 8
        assert np.array_equal(got_map[b][interior, 0], covered[interior].astype(np.float32))
        ok, worst = rel_close(got_map[b][covered, 1], depth[covered], name='shadow edges rendered depth')
        assert ok, (b, worst)


# ---- production sizes -----------------------------------------------------------------------------------------------

PRODUCTION = [
    ('2048^2 shared', False, 2048, 2048),
    ('1024^2 per item', True, 1024, 1024),
    ('2048x512 shared', False, 2048, 512),
    ('512x2048 shared', False, 512, 2048),
]


@pytest.mark.parametrize('case', PRODUCTION, ids=[c[0] for c in PRODUCTION])
@pytest.mark.parametrize('R', [0, 1, 3])
def test_production_sizes(case, R):
    """Three items of 256^2 points with continuous random depths on the benched map sizes, where the coordinate chain
    needs double precision: visibility and all three gradients against the reference."""
    name, per_item, SH, SW = case
    B, N = 3, 256 * 256
    softness = 0.01 if R == 1 else 0.
    p, M, smap = _random_case(B, N, per_item, SH, SW, seed=SH // 7 + SW + R, margin=0.02)
    gout = np.random.default_rng(R).standard_normal((B, N, 1)).astype(np.float32)
    _check(_gpu(p, M, smap, R, softness, gout), _ref(p, M, smap, R, softness, gout, device='cuda'), (name, R))
