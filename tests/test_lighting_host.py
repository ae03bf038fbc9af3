"""CPU: the lighting models' C ABI rejects bad arguments before anything is launched, the routing decision accepts
exactly the plain shapes, and CPU calls run the torch restatement unchanged."""
import ctypes

import numpy as np
import pytest
import torch

DD, SP, DP = 0, 1, 2
CUDA = torch.device('cuda', 0)


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _fwd(L, model=DD, B=1, V=8, C=3, strides=(3, 3, 3), ptrs=None, out=None):
    ok = _p(4096)
    n, p, k, l, lc, cam, s = ptrs if ptrs is not None else [ok] * 7
    sn, sp, sc = strides
    return L.dirt_lighting_forward(model, 1, n, sn, p, sp, k, sc, l, 0, lc, 0, cam, 0, s, 0, ok if out is None else out,
                                   B, V, C, None)


def _bwd(L, model=DD, B=1, V=8, C=3, strides=(3, 3, 3), ptrs=None, grad_out=None, grads=None, ws=None, ws_bytes=1 << 20):
    ok = _p(4096)
    n, p, k, l, lc, cam, s = ptrs if ptrs is not None else [ok] * 7
    sn, sp, sc = strides
    grads = grads if grads is not None else [ok] * 7
    return L.dirt_lighting_backward(model, 0, n, sn, p, sp, k, sc, l, 1, lc, 0, cam, 0, s, 0,
                                    ok if grad_out is None else grad_out, *grads, ok if ws is None else ws, ws_bytes,
                                    B, V, C, None)


def test_lighting_abi_rejects_bad_shapes(L):
    from dirt_b200 import _lib
    for call in (_fwd, _bwd):
        assert call(L, model=3) == _lib.ERR_BAD_SHAPE                  # unknown model
        assert call(L, model=-1) == _lib.ERR_BAD_SHAPE
        assert call(L, B=-1) == _lib.ERR_BAD_SHAPE
        assert call(L, V=-1) == _lib.ERR_BAD_SHAPE
        assert call(L, C=0) == _lib.ERR_BAD_SHAPE
        assert call(L, strides=(-3, 3, 3)) == _lib.ERR_BAD_SHAPE
        assert call(L, strides=(3, 3, -1)) == _lib.ERR_BAD_SHAPE
        assert call(L, B=1 << 30, V=1 << 40) == _lib.ERR_BAD_SHAPE      # element offsets past 2^62
        assert call(L, V=1 << 50, C=1) == _lib.ERR_BAD_SHAPE           # more chunks than the grid holds
        assert L.dirt_last_launch_count() == 0


def test_lighting_workspace_is_a_pure_function_of_the_shapes(L):
    W = L.dirt_lighting_workspace_bytes
    assert W(0, 100, 3) == 0 and W(4, 0, 3) == 0
    assert W(1, 1, 3) == 4 * (7 + 3)
    assert W(64, 512 * 512, 3) == 4 * 64 * 1024 * 10          # 256 points per partial row
    assert W(2, 257, 5) == 4 * 2 * 2 * 12
    assert W(3, 1000, 4) == W(3, 1000, 4)


def test_lighting_abi_with_no_points_launches_nothing(L):
    null = _p(0)
    for B, V in ((0, 8), (3, 0)):
        for model in (DD, SP, DP):
            assert _fwd(L, model, B=B, V=V, ptrs=[null] * 7, out=null) == 0
            assert L.dirt_last_launch_count() == 0
            assert _bwd(L, model, B=B, V=V, ptrs=[null] * 7, grad_out=null, grads=[null] * 7, ws=null, ws_bytes=0) == 0
            assert L.dirt_last_launch_count() == 0


def test_lighting_abi_rejects_null_and_misaligned_pointers(L):
    from dirt_b200 import _lib
    null, ok, odd = _p(0), _p(4096), _p(4098)
    # forward: the inputs each model reads
    needed = {DD: [0, 2, 3, 4], SP: [0, 1, 2, 3, 4, 5, 6], DP: [0, 1, 2, 3, 4]}
    for model, idx in needed.items():
        for k in idx:
            ptrs = [ok] * 7
            ptrs[k] = null
            assert _fwd(L, model, ptrs=ptrs) == _lib.ERR_NULL_POINTER, (model, k)
            assert _bwd(L, model, ptrs=ptrs) == _lib.ERR_NULL_POINTER, (model, k)
            ptrs[k] = odd
            assert _fwd(L, model, ptrs=ptrs) == _lib.ERR_MISALIGNED, (model, k)
            assert _bwd(L, model, ptrs=ptrs) == _lib.ERR_MISALIGNED, (model, k)
        assert _fwd(L, model, out=null) == _lib.ERR_NULL_POINTER
        assert _fwd(L, model, out=odd) == _lib.ERR_MISALIGNED
    # backward: grad_out, every gradient output, the workspace
    assert _bwd(L, SP, grad_out=null) == _lib.ERR_NULL_POINTER
    assert _bwd(L, SP, grad_out=odd) == _lib.ERR_MISALIGNED
    for k in range(7):
        grads = [ok] * 7
        grads[k] = odd
        assert _bwd(L, SP, grads=grads) == _lib.ERR_MISALIGNED, k
    assert _bwd(L, SP, ws=null) == _lib.ERR_NULL_POINTER
    assert _bwd(L, SP, ws=odd) == _lib.ERR_MISALIGNED
    need = L.dirt_lighting_workspace_bytes(1, 8, 3)
    assert _bwd(L, SP, ws_bytes=need - 1) == _lib.ERR_WORKSPACE_TOO_SMALL
    assert L.dirt_last_launch_count() == 0


def test_lighting_route_accepts_the_plain_shapes():
    from dirt_b200.lighting import cuda_route
    dev = [CUDA] * 4
    V3, VC = (1000, 3), (1000, 5)
    # no batch, shared parameters
    r = cuda_route([V3, VC], [((3,), 3), ((5,), 'C')], dev)
    assert r is not None and (r.lead, r.B, r.V, r.C, r.per_item) == ((), 1, 1000, 5, (False, False))
    # [B, V] with per-item and with shared parameters, shininess a scalar or one per item
    r = cuda_route([(4, 100, 3), (4, 100, 3), (4, 100, 2)], [((4, 3), 3), ((2,), 'C'), ((3,), 3), ((4,), 0)], dev)
    assert (r.B, r.V, r.C, r.per_item) == (4, 100, 2, (True, False, False, True))
    r = cuda_route([(4, 100, 3), (4, 100, 3), (4, 100, 2)], [((3,), 3), ((4, 2), 'C'), ((4, 3), 3), ((), 0)], dev)
    assert r.per_item == (False, True, True, False)
    # several leading dimensions; empty batches and empty items
    r = cuda_route([(2, 3, 7, 3), (2, 3, 7, 1)], [((2, 3, 3), 3), ((1,), 'C')], dev)
    assert (r.lead, r.B, r.V, r.C, r.per_item) == ((2, 3), 6, 7, 1, (True, False))
    assert cuda_route([(0, 7, 3), (0, 7, 3)], [((3,), 3), ((0, 3), 'C')], dev).B == 0
    assert cuda_route([(2, 0, 3), (2, 0, 3)], [((3,), 3), ((3,), 'C')], dev).V == 0


def test_lighting_route_refuses_everything_else():
    from dirt_b200.lighting import cuda_route
    dev = [CUDA] * 4
    ok_items = [((3,), 3), ((3,), 'C')]
    assert cuda_route([(100, 3), (100, 3)], ok_items, [torch.device('cpu')] * 4) is None       # CPU
    assert cuda_route([(100, 3), (100, 3)], ok_items, [CUDA, torch.device('cuda', 1)] * 2) is None   # two devices
    assert cuda_route([(100, 3), (100, 3)], ok_items, [CUDA, torch.device('cpu')] * 2) is None
    assert cuda_route([(3,), (3,)], ok_items, dev) is None                                   # no point axis
    assert cuda_route([(100, 4), (100, 3)], ok_items, dev) is None                           # normals not 3 wide
    assert cuda_route([(100, 3), (99, 3)], ok_items, dev) is None                            # V differs
    assert cuda_route([(2, 100, 3), (100, 3)], ok_items, dev) is None                        # colours broadcast
    assert cuda_route([(2, 100, 3), (1, 100, 3)], ok_items, dev) is None
    assert cuda_route([(100, 3), (100, 0)], [((3,), 3), ((0,), 'C')], dev) is None           # C = 0
    assert cuda_route([(100, 3), (100, 3)], [((1, 3), 3), ((3,), 'C')], dev) is None         # light [1, 3] without batch
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((1, 3), 3), ((3,), 'C')], dev) is None   # a broadcast item axis
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((2, 1, 3), 3), ((3,), 'C')], dev) is None
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((3,), 3), ((1,), 'C')], dev) is None     # light colour broadcast
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((3,), 3), ((2, 4), 'C')], dev) is None
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((3,), 3), ((3,), 'C'), ((1,), 0)], dev) is None   # shininess [1]
    assert cuda_route([(2, 100, 3), (2, 100, 3)], [((3,), 3), ((3,), 'C'), ((2, 1), 0)], dev) is None


def _inputs(seed, lead=(2,), V=9, C=3):
    g = torch.Generator().manual_seed(seed)
    n = torch.nn.functional.normalize(torch.randn(lead + (V, 3), generator=g), dim=-1)
    return dict(pos=torch.randn(lead + (V, 3), generator=g), nrm=n, col=torch.rand(lead + (V, C), generator=g),
                ldir=torch.nn.functional.normalize(torch.randn(lead + (3,), generator=g), dim=-1),
                lcol=torch.rand(lead + (C,), generator=g), lpos=torch.randn(lead + (3,), generator=g) * 3,
                cam=torch.randn(lead + (3,), generator=g) * 4, shin=torch.rand(lead, generator=g) * 8)


@pytest.mark.parametrize('double_sided', [True, False])
def test_cpu_calls_return_the_restatement(double_sided):
    from dirt_b200 import lighting
    for lead, C in (((2,), 3), ((), 5), ((2, 3), 1)):
        x = _inputs(len(lead) + C, lead, C=C)
        got = lighting.diffuse_directional(x['nrm'], x['col'], x['ldir'], x['lcol'], double_sided)
        assert torch.equal(got, lighting._diffuse_directional(x['nrm'], x['col'], x['ldir'], x['lcol'], double_sided))
        got = lighting.specular_directional(x['pos'], x['nrm'], x['col'], x['ldir'], x['lcol'], x['cam'], x['shin'],
                                            double_sided)
        want = lighting._specular_directional(x['pos'], x['nrm'], x['col'], x['ldir'], x['lcol'], x['cam'], x['shin'],
                                              double_sided)
        assert torch.equal(got, want)
        got = lighting.diffuse_point(x['pos'], x['nrm'], x['col'], x['lpos'], x['lcol'], double_sided)
        assert torch.equal(got, lighting._diffuse_point(x['pos'], x['nrm'], x['col'], x['lpos'], x['lcol'], double_sided))
    # array-likes and float64 are converted to float32 as before
    x = _inputs(7, (), V=4)
    got = lighting.diffuse_directional(x['nrm'].double().numpy(), x['col'].tolist(), [0., 0., -1.], [1., 1., 1.])
    assert got.dtype == torch.float32
    np.testing.assert_array_equal(got.numpy(), lighting._diffuse_directional(
        x['nrm'], x['col'], torch.tensor([0., 0., -1.]), torch.ones(3)).numpy())


def test_cpu_calls_keep_their_errors():
    from dirt_b200 import lighting
    with pytest.raises(RuntimeError):
        lighting.diffuse_directional(torch.zeros(5, 3), torch.zeros(5, 3), torch.zeros(4), torch.zeros(3))
    with pytest.raises(RuntimeError):
        lighting.diffuse_point(torch.zeros(5, 3), torch.zeros(5, 3), torch.zeros(4, 3), torch.zeros(3), torch.zeros(3))
