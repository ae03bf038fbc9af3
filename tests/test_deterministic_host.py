"""CPU: the deterministic backward pass's C ABI rejects bad arguments before anything is enqueued, its scratch size is a
function of the shapes alone, and rasterise_backward_raw follows torch.use_deterministic_algorithms."""
import ctypes

import pytest
import torch


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _call(L, B=2, H=16, W=16, C=3, V=8, F=4, groups=None, flags=0, ids=4096, ws=4096, ws_bytes=1 << 30,
          scratch=4096, scratch_bytes=1 << 30, **ptrs):
    p = dict(vertices=4096, faces=4096, pixels=4096, grad_pixels=4096, grad_background=4096, grad_vertices=4096,
             grad_vertex_colors=4096)
    p.update(ptrs)
    g = (ctypes.c_int * len(groups))(*groups) if groups else None
    return L.dirt_rasterise_backward_deterministic(
        _p(p['vertices']), _p(p['faces']), _p(p['pixels']), _p(p['grad_pixels']), _p(ids), _p(p['grad_background']),
        _p(p['grad_vertices']), _p(p['grad_vertex_colors']), B, H, W, C, V, F, g, len(groups) if groups else 0, 0, flags,
        _p(ws), ws_bytes, _p(scratch), scratch_bytes, None)


def test_rejects_bad_arguments_before_launching(L):
    from dirt_b200 import _lib
    cases = [
        (dict(B=-1), _lib.ERR_BAD_SHAPE), (dict(H=0), _lib.ERR_BAD_SHAPE), (dict(C=0), _lib.ERR_BAD_SHAPE),
        (dict(flags=8), _lib.ERR_BAD_SHAPE), (dict(flags=-1), _lib.ERR_BAD_SHAPE),
        (dict(B=3, F=(1 << 31) // 9 + 1, H=1, W=1), _lib.ERR_BAD_SHAPE),   # corner ids 3*B*F past int32
        (dict(V=(1 << 24) + 1), _lib.ERR_TOO_MANY_VERTICES),
        (dict(groups=[3, 3]), _lib.ERR_BAD_CHANNEL_GROUPS), (dict(groups=[2, 1]), _lib.ERR_BAD_CHANNEL_GROUPS),
        (dict(C=4, groups=[1, 1, 1]), _lib.ERR_BAD_CHANNEL_GROUPS),
        (dict(grad_pixels=0), _lib.ERR_NULL_POINTER), (dict(pixels=0), _lib.ERR_NULL_POINTER),
        (dict(grad_background=0), _lib.ERR_NULL_POINTER), (dict(vertices=0), _lib.ERR_NULL_POINTER),
        (dict(faces=0), _lib.ERR_NULL_POINTER), (dict(grad_vertices=0), _lib.ERR_NULL_POINTER),
        (dict(grad_vertex_colors=0), _lib.ERR_NULL_POINTER), (dict(ws=0), _lib.ERR_NULL_POINTER),
        (dict(scratch=0), _lib.ERR_NULL_POINTER),
        (dict(vertices=4104), _lib.ERR_MISALIGNED), (dict(grad_vertices=4104), _lib.ERR_MISALIGNED),
        (dict(pixels=4098), _lib.ERR_MISALIGNED), (dict(ws=4224), _lib.ERR_MISALIGNED),
        (dict(scratch=4224), _lib.ERR_MISALIGNED),
        (dict(ws_bytes=1024), _lib.ERR_WORKSPACE_TOO_SMALL),
        (dict(scratch_bytes=L.dirt_rasterise_backward_deterministic_bytes(2, 16, 16, 3, 8, 4) - 1), _lib.ERR_WORKSPACE_TOO_SMALL),
    ]
    for kw, rc in cases:
        assert _call(L, **kw) == rc, kw
        assert L.dirt_last_launch_count() == 0
    # pointers a flag makes unnecessary
    assert _call(L, flags=2, pixels=0, scratch=0) == _lib.ERR_NULL_POINTER   # still needs the scratch
    assert _call(L, flags=4, grad_background=0, scratch=0) == _lib.ERR_NULL_POINTER
    # an empty batch is a no-op
    assert _call(L, B=0, scratch=0, ws=0) == 0
    assert L.dirt_last_launch_count() == 0


def test_scratch_size_is_a_function_of_the_shapes(L):
    size = L.dirt_rasterise_backward_deterministic_bytes
    assert size(0, 16, 16, 3, 8, 4) == 0
    assert size(-1, 16, 16, 3, 8, 4) == 0 and size(1, 0, 16, 3, 8, 4) == 0
    base = (4, 32, 48, 3, 100, 60)
    s0 = size(*base)
    assert s0 > 0 and s0 % 256 == 0 and size(*base) == s0
    for i in range(6):
        bigger = list(base)
        bigger[i] *= 2
        assert size(*bigger) >= s0, bigger
    # per pixel at least the codes (C planes) and dL/dx, dL/dy; per face a box and the float64 partials
    B, H, W, C, V, F = base
    assert s0 >= B * H * W * (C + 8) + B * F * (16 + 3 * (3 + C) * 8)
    # the largest shapes the workspace size functions accept: no overflow, still monotone
    for shape in ((1, 1 << 15, 1 << 15, 384, 1 << 24, (1 << 31) - 1), (255, 1 << 15, 1 << 15, 384, 1 << 24, 1),
                  ((1 << 31) - 1, 8, 8, 384, 1 << 24, 1)):
        assert L.dirt_workspace_bytes(*shape) > 0, shape
        big = size(*shape)
        assert big >= L.dirt_workspace_bytes(*shape) // 4, shape   # at least a byte per pixel and channel, no wrap-round
        smaller = list(shape)
        smaller[0] = max(1, shape[0] // 2)
        assert size(*smaller) <= big, shape


@pytest.fixture
def deterministic_algorithms():
    before = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(before)


def _route(monkeypatch, **kw):
    """Which entry point rasterise_backward_raw calls (the library calls are replaced by recorders)."""
    from dirt_b200 import _lib
    from dirt_b200 import rasterise_ops as ops
    called = []

    class Fake:
        def __getattr__(self, name):
            def f(*args):
                called.append(name)
                return 1024
            return f

    monkeypatch.setattr(_lib, 'lib', lambda: Fake())
    monkeypatch.setattr(_lib, 'check', lambda rc, what: None)
    monkeypatch.setattr(ops, '_stream_ptr', lambda device: None)

    class Dev:
        def __init__(self, *a):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

    monkeypatch.setattr(ops.torch.cuda, 'device', Dev)
    v = torch.zeros(1, 3, 4)
    f = torch.zeros(1, 1, 3, dtype=torch.int32)
    px = torch.zeros(1, 4, 4, 3)
    ops.rasterise_backward_raw(v, f, px, px, **kw)
    return [c for c in called if c.startswith('dirt_rasterise_backward')]


def test_routing_follows_torch_deterministic_algorithms(monkeypatch, deterministic_algorithms):
    det = ['dirt_rasterise_backward_deterministic_bytes', 'dirt_rasterise_backward_deterministic']
    torch.use_deterministic_algorithms(False)
    assert _route(monkeypatch) == ['dirt_rasterise_backward_ex']
    assert _route(monkeypatch, deterministic=True) == det
    torch.use_deterministic_algorithms(True)
    assert _route(monkeypatch) == det
    assert _route(monkeypatch, deterministic=False) == ['dirt_rasterise_backward_ex']
