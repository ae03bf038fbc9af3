"""GPU: the mesh kernels of csrc/normals.cu bit for bit against tests/mesh_order.py, their float32 restatement.

1. The corner adjacency read back from the workspace (offsets at 0, inc at round_up(4(V+1), 256), then the build's
   counts and unsorted ids) after dirt_normals_forward and dirt_laplacian_forward, at row counts around multiples of the
   one-CTA scan's 1024 threads and at the Laplacian benchmark's V, with invalid indices; and the deterministic
   rasteriser backward pass's adjacency of B face tables, read from its scratch (det_records.read_scratch).
2. Every output and gradient of the vertex normals (both modes), the vertex tangents and the Laplacian (both modes),
   compared as int32 views (NaN only as NaN), on the existing suites' meshes and on the degenerate ones those suites
   leave out: faces naming a vertex twice or three times, collinear and zero-area faces, reversed and duplicated faces,
   non-manifold edges, isolated vertices, a folded sheet, cotangent slivers; and the tangents' degenerate uvs, mirrored
   uvs, a tangent along the normal, a zero normal, and each gradient asked for alone.
3. The row-sum boundary: rows of exactly 32 and 33 corners, a warp of 32 long rows, warps straddling two items with long
   rows on both sides and a partly empty last warp; each item alone gives the bits it gets inside a batch.
4. The edge lengths and normal consistency (both face passes, both vertex passes) on the same meshes, on
   test_gpu_edge_terms.py's degenerate mesh (duplicated, reversed, non-manifold, repeated-index and zero-area faces)
   and on a fan of 5000 faces, whose partner search scans the rim rows and never the hub's.
5. The same against the small-grid build, whose launches run many grid-stride rounds."""
import ctypes

import numpy as np
import pytest
import torch

import det_records as dr
import mesh_order as mo
import variant_builds

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _same(got, want, what):
    if isinstance(got, torch.Tensor):
        got = got.detach().cpu().numpy()
    msg = mo.first_difference(got, want)
    assert msg is None, '%s: %s' % (what, msg)


def _round256(n):
    return (n + 255) // 256 * 256


# ---- 1. the adjacency, exactly ------------------------------------------------------------------------------------------

def read_workspace(buf, V, F):
    """carve_normals_workspace's blocks after a forward call: offsets [V + 1], inc [3F], counts [V], unsorted [3F]."""
    buf = np.asarray(buf, np.uint8)
    o_inc = _round256(4 * (V + 1))
    o_counts = o_inc + _round256(12 * F)
    o_unsorted = o_counts + _round256(4 * V)
    view = lambda o, n: buf[o:o + 4 * n].view(np.int32)
    return dict(offsets=view(0, V + 1), inc=view(o_inc, 3 * F), counts=view(o_counts, V),
                unsorted=view(o_unsorted, 3 * F))


def check_adjacency(got, offsets, inc, what):
    n = int(offsets[-1])
    assert np.array_equal(got['offsets'], offsets), what + ': offsets'
    assert np.array_equal(got['inc'][:n], inc), what + ': inc'
    assert not got['counts'].any(), what + ': counts not back to 0'
    rows = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    u = got['unsorted'][:n]
    order = np.lexsort((u, rows))
    assert np.array_equal(u[order], inc), what + ': a row of unsorted ids is not a permutation of its row of inc'


def _adjacency_faces(V, seed):
    """Random faces over V vertices, a hub of 40 corners when V allows, and faces with invalid indices -1, V and
    2^31 - 1; for the benchmark's V the faces of its uv-sphere (1024 x 512: poles of valence 1024)."""
    from dirt_b200 import scenes
    if V >= 1024 * 511 + 1:
        _, f = scenes.uv_sphere(1024, 512)
        # at V = 1024*511 + 1 the faces of the last pole name vertex V: all of them are left out
        return np.concatenate([f, [[0, 1, -1], [V, 0, 1], [2, (1 << 31) - 1, 3]]]).astype(np.int32)
    r = np.random.default_rng(seed)
    f = r.integers(0, V, (2 * V + 40, 3))
    if V > 3:
        f[:40, 0] = V // 2
    bad = r.choice(len(f), min(len(f), 30), replace=False)
    f[bad, r.integers(0, 3, len(bad))] = r.choice([-1, V, (1 << 31) - 1], len(bad))
    return f.astype(np.int32)


ROW_COUNTS = [1, 31, 32, 1023, 1024, 1025, 2047, 2049, 1024 * 511 + 1, 1024 * 511 + 2]


@pytest.mark.parametrize('V', ROW_COUNTS)
def test_adjacency_read_back_from_the_workspace(cuda_lib, V):
    L = cuda_lib
    f = _adjacency_faces(V, V)
    F = len(f)
    offsets, inc = mo.adjacency(f, V)
    x = torch.randn((V, 3), generator=torch.Generator(device=DEV).manual_seed(V), device=DEV)
    faces = torch.tensor(f, device=DEV)
    out = torch.empty((V, 3), device=DEV)
    for name, call, size in (('normals', L.dirt_normals_forward, L.dirt_normals_workspace_bytes),
                             ('laplacian', L.dirt_laplacian_forward, L.dirt_laplacian_workspace_bytes)):
        n = int(size(1, V, F))
        ws = torch.full((n,), 0xA5, dtype=torch.uint8, device=DEV)
        assert call(0, _p(x), 3, _p(faces), _p(out), _p(ws), n, 1, V, F, _stream()) == 0
        torch.cuda.synchronize()
        check_adjacency(read_workspace(ws.cpu().numpy(), V, F), offsets, inc, '%s V=%d' % (name, V))


def _mesh_node(t):
    """The mesh op's autograd node behind t (its context holds the workspace)."""
    todo = [t.grad_fn]
    while todo:
        node = todo.pop()
        if node is not None and hasattr(node, 'workspace'):
            return node
        todo += [n for n, _ in (node.next_functions if node is not None else ())]
    raise AssertionError('no mesh node')


def test_int64_faces_clamp_into_invalid_indices(cuda_lib):
    """int64 indices past int32 are clamped to -1 or 2^31 - 1, so they are left out like any invalid index: the
    workspace's adjacency, the outputs and the gradients are those of the faces without them."""
    from dirt_b200 import lighting
    v, f = mo.icosphere()
    V = len(v)
    bad = f.astype(np.int64)
    for j, value in enumerate([(1 << 32) + 3, (1 << 32) + V - 1, -(1 << 32) + 2, 1 << 31, 1 << 40, -(1 << 40), V, -1]):
        bad[5 + 37 * j, j % 3] = value
    P = v[None]
    x = torch.tensor(P, device=DEV).requires_grad_(True)
    out = lighting.vertex_normals(x, torch.tensor(bad, device=DEV))
    node = _mesh_node(out)
    offsets, inc = mo.adjacency(bad, V)
    check_adjacency(read_workspace(node.workspace.cpu().numpy(), V, len(f)), offsets, inc, 'int64 faces')
    g = torch.randn(out.shape, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    _same(out, mo.normals_forward(P, bad), 'normals, int64 faces')
    out.backward(g)
    _same(x.grad, mo.normals_backward(P, bad, g.cpu().numpy()), 'normals grad, int64 faces')


def _det_scene(B, V, F, seed):
    """A random soup of B items whose face tables differ per item, each with a hub of 40 corners."""
    from dirt_b200 import scenes
    s = scenes.random_soup(batch=B, width=40, height=24, n_faces=F, channels=3, seed=seed)
    r = np.random.default_rng(seed)
    V0 = s['vertices'].shape[1]
    assert V0 == V
    faces = np.stack([np.stack([r.permutation(V)[:3] for _ in range(F)]) for _ in range(B)])
    faces[:, :40, 1] = np.arange(B)[:, None] + 3
    s['faces'] = faces.astype(np.int32)
    return s


@pytest.mark.parametrize('flags', [0, dr.SHARED_GEOMETRY])
def test_deterministic_backward_adjacency(cuda_lib, flags):
    """The deterministic rasteriser backward pass builds one adjacency over its B face tables (items = B, face_stride
    = 3F), whether or not the geometry is shared: offsets, counts and inc read from its scratch."""
    from test_gpu_paths import abi_forward
    L = cuda_lib
    B, F, C, H, W = 3, 70, 3, 24, 40
    V = F + 2
    s = _det_scene(B, V, F, 11)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in s.items()}
    pixels = torch.empty_like(t['background'])
    ids = torch.empty((B, H, W), dtype=torch.int32, device=DEV)
    abi_forward(L, t['background'], t['vertices'], t['vertex_colors'], t['faces'], pixels, ids)
    gp = torch.randn(pixels.shape, generator=torch.Generator(device=DEV).manual_seed(12), device=DEV)
    lead = () if flags & dr.SHARED_GEOMETRY else (B,)
    gb, gv, gc = torch.empty_like(pixels), torch.empty(lead + (V, 4), device=DEV), torch.empty(lead + (V, C), device=DEV)
    n = max(int(L.dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F)), 256)
    scratch = torch.full((n,), 0xA5, dtype=torch.uint8, device=DEV)
    ws = torch.empty(int(L.dirt_workspace_bytes(B, H, W, C, V, F)), dtype=torch.uint8, device=DEV)
    groups = (ctypes.c_int * 1)(C)
    rc = L.dirt_rasterise_backward_deterministic(_p(t['vertices']), _p(t['faces']), _p(pixels), _p(gp), _p(ids), _p(gb),
                                                 _p(gv), _p(gc), B, H, W, C, V, F, groups, 1, 0, flags, _p(ws),
                                                 ws.numel(), _p(scratch), n, _stream())
    assert rc == 0, L.dirt_error_string(rc)
    got = dr.read_scratch(scratch.cpu().numpy(), B, H, W, C, V, F)
    offsets, inc = mo.adjacency(s['faces'], V, items=B, face_stride=3 * F)
    assert (np.diff(offsets) > mo.LONG_ROW).sum() == B
    check_adjacency(got, offsets, inc, 'deterministic backward flags=%d' % flags)


# ---- 2, 3. every output and gradient, bit for bit ----------------------------------------------------------------------

MESHES = {
    'icosphere': (mo.icosphere, 2), 'uv_sphere': (mo.uv_sphere, 2), 'fan': (mo.fan, 1), 'grid': (mo.grid, 2),
    'odd': (mo.odd, 2), 'degenerate': (mo.degenerate, 2), 'folded': (mo.folded, 2), 'slivers': (mo.slivers, 2),
    'rows_32_33': (mo.rows_32_33, 2), 'full_warp': (mo.full_warp, 2), 'straddle': (mo.straddle, 3),
}


def _items(v, B, seed):
    """[B, V, 4] float32 on the device, every other item of a batch of 2B (strided items, row stride 4)."""
    g = np.random.default_rng(seed)
    P = v[None] * (1. + 0.1 * g.random((2 * B, 1, 1))) + 0.1 * g.standard_normal((2 * B, 1, 3))
    x = np.concatenate([P, 1. + g.random(P.shape[:-1] + (1,))], -1).astype(np.float32)
    return torch.tensor(x, device=DEV)[::2]


def _grad(shape, seed):
    return torch.randn(shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)


def check_normals_and_laplacian(v, f, B, seed, what):
    """Forward and backward of the normals and the Laplacian, both modes of each, on B strided items [B, V, 4];
    -> ({op: (out, grad)} as numpy, the items)."""
    from dirt_b200 import lighting, mesh
    x = _items(v, B, seed)
    P = x[..., :3].cpu().numpy()
    faces = torch.tensor(f, device=DEV)
    g = _grad(x.shape[:-1] + (3,), seed + 1)
    gn = g.cpu().numpy()
    ops = {'normals': (lambda t: lighting.vertex_normals(t, faces), lambda: mo.normals_forward(P, f),
                       lambda: mo.normals_backward(P, f, gn)),
           'pre-split': (lambda t: lighting.vertex_normals_pre_split(t, faces),
                         lambda: mo.normals_forward(P, f, mo.PRE_SPLIT),
                         lambda: mo.normals_backward(P, f, gn, mo.PRE_SPLIT))}
    for mode, m in (('uniform', mo.UNIFORM), ('cotangent', mo.COTANGENT)):
        ops['laplacian ' + mode] = (lambda t, mode=mode: mesh.laplacian(t, faces, mode),
                                    lambda m=m: mo.laplacian_forward(P, f, m),
                                    lambda m=m: mo.laplacian_backward(P, f, gn, m))
    results = {}
    for name, (op, fwd, bwd) in ops.items():
        leaf = x.detach().clone().requires_grad_(True)
        out = op(leaf)
        out.backward(g)
        _same(out, fwd(), '%s %s forward' % (what, name))
        _same(leaf.grad[..., :3], bwd(), '%s %s grad_vertices' % (what, name))
        assert not leaf.grad[..., 3].any()
        results[name] = (out.detach().cpu().numpy(), leaf.grad.cpu().numpy())
    return results, x


@pytest.mark.parametrize('name', sorted(MESHES))
def test_normals_and_laplacian_bit_for_bit(cuda_lib, name):
    fixture, B = MESHES[name]
    v, f = fixture()
    batch, x = check_normals_and_laplacian(v, f, B, 20, name)
    if B > 1:
        # each item alone gives the bits it gets inside the batch
        from dirt_b200 import lighting, mesh
        faces = torch.tensor(f, device=DEV)
        g = _grad(x.shape[:-1] + (3,), 21)
        ops = {'normals': lambda t: lighting.vertex_normals(t, faces),
               'pre-split': lambda t: lighting.vertex_normals_pre_split(t, faces),
               'laplacian uniform': lambda t: mesh.laplacian(t, faces, 'uniform'),
               'laplacian cotangent': lambda t: mesh.laplacian(t, faces, 'cotangent')}
        for op_name, op in ops.items():
            leaf = x.detach().clone().requires_grad_(True)
            out = op(leaf)
            out.backward(g)
            for b in range(B):
                one = x[b].detach().clone().requires_grad_(True)
                o = op(one)
                o.backward(g[b])
                _same(o, out[b].detach().cpu().numpy(), '%s %s item %d alone: forward' % (name, op_name, b))
                _same(one.grad, leaf.grad[b].cpu().numpy(), '%s %s item %d alone: grad' % (name, op_name, b))


def test_kinks_bit_for_bit(cuda_lib):
    """Integer coordinates: a collinear face, a face naming a vertex twice and a face with its reversed copy; the
    normals' 1e24-scale gradients and the Laplacian's zero-area faces (the c.nn == 0 branch)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 1, 0], [4, 2, 1], [0, 5, 0], [1, 5, 2], [0, 6, 3]], np.float32)
    f = np.array([[0, 1, 2], [3, 3, 4], [5, 6, 7], [5, 7, 6]], np.int32)
    from dirt_b200 import lighting, mesh
    x = torch.tensor(v, device=DEV)[None]
    faces = torch.tensor(f, device=DEV)
    g = torch.tensor(np.random.default_rng(12).integers(-3, 4, (1, 8, 3)), dtype=torch.float32, device=DEV)
    P, gn = v[None], g.cpu().numpy()
    for name, op, fwd, bwd in (
            ('normals', lambda t: lighting.vertex_normals(t, faces), mo.normals_forward(P, f),
             mo.normals_backward(P, f, gn)),
            ('laplacian cotangent', lambda t: mesh.laplacian(t, faces, 'cotangent'),
             mo.laplacian_forward(P, f, mo.COTANGENT), mo.laplacian_backward(P, f, gn, mo.COTANGENT))):
        leaf = x.clone().requires_grad_(True)
        out = op(leaf)
        out.backward(g)
        _same(out, fwd, 'kinks %s forward' % name)
        _same(leaf.grad, bwd, 'kinks %s grad' % name)
    assert np.abs(mo.normals_backward(P, f, gn)).max() > 1e23


# ---- the tangents ---------------------------------------------------------------------------------------------------------

def _tangent_meshes():
    v, uv, f, n = mo.tangent_cases()
    out = {'cases': (v, uv, f, n)}
    for name, fixture in (('fan', lambda: mo.fan(3000)), ('straddle', mo.straddle), ('full_warp', mo.full_warp),
                          ('degenerate', mo.degenerate)):
        v, f = fixture()
        out[name] = (v, mo.uv_for(v), f, None)
    v, uv, f = mo.seamed_sphere(224, 112)
    out['seamed_sphere'] = (v, uv, f, None)
    return out


TANGENT_MESHES = ['cases', 'fan', 'straddle', 'full_warp', 'degenerate', 'seamed_sphere']
WANTS = {'all': (True, True, True), 'vertices': (True, False, False), 'uvs': (False, True, False),
         'normals': (False, False, True)}


@pytest.mark.parametrize('want', sorted(WANTS))
@pytest.mark.parametrize('name', TANGENT_MESHES)
def test_tangents_bit_for_bit(cuda_lib, name, want):
    check_tangents(name, want)


def check_tangents(name, want):
    """The tangents of 3 items with per-item uvs (one item with the fixture's own uvs) and their gradients, only those
    of `want` asked for; with want = 'all', the forward with shared uvs too."""
    from dirt_b200 import lighting
    v, uv, f, n = _tangent_meshes()[name]
    B = 3
    x = _items(v, B, 30)
    P = x[..., :3].cpu().numpy()
    r = np.random.default_rng(31)
    U = (uv[None] + 0.01 * r.standard_normal((B,) + uv.shape)).astype(np.float32)
    U[1] = uv   # one item keeps the fixture's exact (degenerate) uvs
    if n is None:
        N = mo.normals_forward(P, f) + 0.05 * r.standard_normal(P.shape)
    else:
        N = np.broadcast_to(n, P.shape)
    N = np.ascontiguousarray(N, np.float32)
    faces = torch.tensor(f, device=DEV)
    uvs, normals = torch.tensor(U, device=DEV), torch.tensor(N, device=DEV)
    wv, wu, wn = WANTS[want]
    xl, ul, nl = x.clone().requires_grad_(wv), uvs.clone().requires_grad_(wu), normals.clone().requires_grad_(wn)
    out = lighting.vertex_tangents(xl, ul, faces, nl)
    _same(out, mo.tangents_forward(P, U, N, f), '%s tangents forward' % name)
    g = _grad(out.shape, 32)
    out.backward(g)
    gp, gu, gn = mo.tangents_backward(P, U, N, f, g.cpu().numpy(), wv, wu, wn)
    if wv:
        _same(xl.grad[..., :3], gp, '%s tangents grad_vertices' % name)
    if wu:
        _same(ul.grad, gu, '%s tangents grad_uvs' % name)
    if wn:
        _same(nl.grad, gn, '%s tangents grad_normals' % name)
    if want == 'all':
        # shared uvs: the same tangents as per-item copies of them
        shared = lighting.vertex_tangents(x, torch.tensor(uv, device=DEV), faces, normals)
        _same(shared, mo.tangents_forward(P, uv, N, f), '%s tangents forward, shared uvs' % name)


# ---- 4. the edge terms -----------------------------------------------------------------------------------------------------

def _edge_meshes():
    from test_gpu_edge_terms import _degenerate
    out = dict(MESHES)
    out['edge_degenerate'] = (_degenerate, 2)
    out['fan_5000'] = (lambda: mo.fan(5000), 3)
    return out


EDGE_MESHES = sorted(MESHES) + ['edge_degenerate', 'fan_5000']


def check_edge_terms(v, f, B, seed, what):
    """Forward and backward of both edge terms on B strided items [B, V, 4]."""
    from dirt_b200 import mesh
    x = _items(v, B, seed)
    P = x[..., :3].cpu().numpy()
    faces = torch.tensor(f, device=DEV)
    g = _grad((B, len(f), 3), seed + 1)
    for name, m in (('edge_lengths', mo.LENGTH), ('normal_consistency', mo.CONSISTENCY)):
        leaf = x.detach().clone().requires_grad_(True)
        out = getattr(mesh, name)(leaf, faces)
        out.backward(g)
        _same(out, mo.edge_terms_forward(P, f, m), '%s %s forward' % (what, name))
        _same(leaf.grad[..., :3], mo.edge_terms_backward(P, f, g.cpu().numpy(), m), '%s %s grad_vertices' % (what, name))
        assert not leaf.grad[..., 3].any()


@pytest.mark.parametrize('name', EDGE_MESHES)
def test_edge_terms_bit_for_bit(cuda_lib, name):
    fixture, B = _edge_meshes()[name]
    v, f = fixture()
    check_edge_terms(v, f, B, 50, name)


# ---- 5. the small-grid build ------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def small(cuda_lib, tmp_path_factory):
    return variant_builds.small_grid_library(tmp_path_factory)


@pytest.mark.parametrize('name', ['degenerate', 'straddle', 'full_warp', 'uv_sphere'])
def test_small_grid_build_bit_for_bit(cuda_lib, small, name):
    """DIRT_NORMALS_MAX_BLOCKS = 3: every vertex pass and adjacency kernel runs many grid-stride rounds."""
    from dirt_b200 import _lib
    fixture, B = MESHES[name]
    v, f = fixture()
    with pytest.MonkeyPatch.context() as m:
        m.setattr(_lib, 'lib', lambda: small)
        check_normals_and_laplacian(v, f, max(B, 3), 40, name + ' (small grid)')
        check_tangents('degenerate' if name == 'degenerate' else 'straddle', 'all')


@pytest.mark.parametrize('name', ['edge_degenerate', 'straddle', 'fan_5000', 'uv_sphere'])
def test_small_grid_build_edge_terms_bit_for_bit(cuda_lib, small, name):
    """DIRT_NORMALS_MAX_BLOCKS = 3: the edge terms' face and vertex passes run many grid-stride rounds."""
    from dirt_b200 import _lib
    fixture, B = _edge_meshes()[name]
    v, f = fixture()
    with pytest.MonkeyPatch.context() as m:
        m.setattr(_lib, 'lib', lambda: small)
        check_edge_terms(v, f, max(B, 3), 60, name + ' (small grid)')
