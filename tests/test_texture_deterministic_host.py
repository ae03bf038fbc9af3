"""CPU: the deterministic texture backward pass's C ABI rejects bad arguments before anything is enqueued, its scratch
size is a function of the shapes alone, sample_texture's backward follows torch.use_deterministic_algorithms, and the
numpy restatement of its summation order agrees with exact sums."""
import ctypes
import math

import numpy as np
import pytest
import torch

import texture_det_order as order


@pytest.fixture(scope='module')
def L():
    from dirt_b200 import build, _lib
    build.build()
    return _lib.lib()


def _p(x):
    return ctypes.c_void_p(x)


def _call(L, TB=1, TH=8, TW=8, C=3, B=2, N=100, mode=0, scratch=4096, scratch_bytes=1 << 30, **ptrs):
    p = dict(texture=4096, indices=4096, grad_out=4096, grad_texture=4096, grad_indices=4096)
    p.update(ptrs)
    return L.dirt_texture_sample_backward_deterministic(
        _p(p['texture']), _p(p['indices']), _p(p['grad_out']), _p(p['grad_texture']), _p(p['grad_indices']), TB, TH, TW, C,
        B, N, mode, _p(scratch), scratch_bytes, None)


def test_rejects_bad_arguments_before_launching(L):
    from dirt_b200 import _lib
    size = L.dirt_texture_sample_backward_deterministic_bytes
    cases = [
        (dict(TH=0), _lib.ERR_BAD_SHAPE), (dict(TW=0), _lib.ERR_BAD_SHAPE), (dict(C=0), _lib.ERR_BAD_SHAPE),
        (dict(B=-1), _lib.ERR_BAD_SHAPE), (dict(N=-1), _lib.ERR_BAD_SHAPE), (dict(TB=2, B=3), _lib.ERR_BAD_SHAPE),
        (dict(mode=2), _lib.ERR_BAD_SHAPE),
        (dict(B=1, N=1 << 31), _lib.ERR_BAD_SHAPE),                        # lookup ids past int32
        (dict(B=2, N=1 << 30), _lib.ERR_BAD_SHAPE),
        (dict(TH=1 << 16, TW=(1 << 15)), _lib.ERR_BAD_SHAPE),             # TB*TH*TW = 2^31 - 1 + 1: no room for the sentinel
        (dict(TH=(1 << 31) - 1, TW=1), _lib.ERR_BAD_SHAPE),
        (dict(indices=0), _lib.ERR_NULL_POINTER), (dict(grad_out=0), _lib.ERR_NULL_POINTER),
        (dict(texture=0), _lib.ERR_NULL_POINTER),                          # bilinear grad_indices reads the texture
        (dict(scratch=0), _lib.ERR_NULL_POINTER),
        (dict(texture=4098), _lib.ERR_MISALIGNED), (dict(indices=4098), _lib.ERR_MISALIGNED),
        (dict(grad_out=4098), _lib.ERR_MISALIGNED), (dict(grad_texture=4098), _lib.ERR_MISALIGNED),
        (dict(grad_indices=4098), _lib.ERR_MISALIGNED), (dict(scratch=4224), _lib.ERR_MISALIGNED),
        (dict(scratch_bytes=size(1, 8, 8, 3, 2, 100, 0) - 1), _lib.ERR_WORKSPACE_TOO_SMALL),
        (dict(scratch_bytes=0), _lib.ERR_WORKSPACE_TOO_SMALL),
    ]
    for kw, rc in cases:
        assert _call(L, **kw) == rc, kw
        assert L.dirt_last_launch_count() == 0
    # the largest shapes the limits allow pass validation (a NULL scratch is the first thing that fails)
    assert _call(L, B=1, N=(1 << 31) - 1, scratch=0) == _lib.ERR_NULL_POINTER
    assert _call(L, TH=1 << 16, TW=(1 << 15) - 1, scratch=0) == _lib.ERR_NULL_POINTER
    # nothing to sort: the scratch may be NULL
    assert _call(L, B=0, scratch=0, texture=0, indices=0, grad_out=0, grad_texture=0, grad_indices=0) == 0
    assert _call(L, N=0, scratch=0, texture=0, indices=0, grad_out=0, grad_texture=0, grad_indices=0) == 0
    assert L.dirt_last_launch_count() == 0


def test_scratch_size_is_a_function_of_the_shapes(L):
    size = L.dirt_texture_sample_backward_deterministic_bytes
    assert size(1, 8, 8, 3, 0, 100, 0) == 0 and size(1, 8, 8, 3, 2, 0, 0) == 0
    assert size(1, 0, 8, 3, 2, 100, 0) == 0 and size(1, 8, 8, 3, 2, 100, 2) == 0
    assert size(1, 8, 8, 3, 1, 1 << 31, 0) == 0 and size(1, 1 << 16, 1 << 15, 3, 1, 8, 0) == 0
    base = (4, 32, 48, 3, 4, 5000, 0)
    s0 = size(*base)
    assert s0 > 0 and s0 % 256 == 0 and size(*base) == s0
    for i in (1, 2, 3, 5):
        bigger = list(base)
        bigger[i] *= 2
        assert size(*bigger) > s0, bigger
    assert size(1, 32, 48, 3, 4, 5000, 0) < s0                      # per-item textures need more offsets
    assert size(*base[:-1], 1) <= s0                                # nearest has one term per lookup, not four
    # at least the double-buffered keys and ids and one offset per texel
    TB, TH, TW, C, B, N, _ = base
    assert s0 >= 16 * B * N + 4 * (TB * TH * TW + 2)
    # the largest shapes: no overflow, still monotone
    big = size(1, 1 << 15, (1 << 16) - 1, 8, 1, (1 << 31) - 1, 0)
    assert big >= 16 * ((1 << 31) - 1) and big >= size(1, 1 << 15, (1 << 16) - 1, 8, 1, 1 << 30, 0)


@pytest.fixture
def deterministic_algorithms():
    before = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(before)


def _route(monkeypatch, want=(True, True), rc=0):
    """The entry points one sample_texture backward pass calls (the library calls are replaced by recorders that return
    `rc`, and 1024 for the size query)."""
    from dirt_b200 import _lib
    from dirt_b200 import texture as tx
    called = []

    class Fake:
        def __getattr__(self, name):
            def f(*args):
                called.append(name)
                return 1024 if name.endswith('_bytes') else (rc if name.endswith('deterministic') else 0)
            return f

    class Dev:
        def __init__(self, *a):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

    monkeypatch.setattr(_lib, 'lib', lambda: Fake())
    monkeypatch.setattr(tx, '_stream_ptr', lambda device: None)
    monkeypatch.setattr(tx.torch.cuda, 'device', Dev)
    tex = torch.zeros(1, 4, 4, 3, requires_grad=want[0])
    idx = torch.zeros(1, 5, 2, requires_grad=want[1])
    tx._SampleTexture.apply(tex, idx, _lib.TEXTURE_BILINEAR, (1, 5, 3)).sum().backward()
    return [c for c in called if c.startswith('dirt_texture_sample_backward')]


def test_routing_follows_torch_deterministic_algorithms(monkeypatch, deterministic_algorithms):
    det = ['dirt_texture_sample_backward_deterministic_bytes', 'dirt_texture_sample_backward_deterministic']
    torch.use_deterministic_algorithms(False)
    assert _route(monkeypatch) == ['dirt_texture_sample_backward']
    assert _route(monkeypatch, want=(True, False)) == ['dirt_texture_sample_backward']
    torch.use_deterministic_algorithms(True)
    assert _route(monkeypatch) == det
    assert _route(monkeypatch, want=(True, False)) == det
    # grad_indices alone is already deterministic: the default entry
    assert _route(monkeypatch, want=(False, True)) == ['dirt_texture_sample_backward']


def test_shapes_beyond_the_limits_raise_naming_the_flag(monkeypatch, deterministic_algorithms):
    from dirt_b200 import _lib
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match=r'torch\.use_deterministic_algorithms'):
        _route(monkeypatch, rc=_lib.ERR_BAD_SHAPE)


def test_restated_order_agrees_with_exact_sums():
    """The restatement's tree against math.fsum of the same terms, within one fp32 ulp, on sequences from empty to
    many chunks long."""
    rng = np.random.default_rng(0)
    lengths = [0, 1, 2, 31, 32, 33, 100, 4095, 4096, 4097, 8192, 3 * 4096 + 17, 40000]
    texel = np.concatenate([np.full(n, k) for k, n in enumerate(lengths)]).astype(np.int64)
    terms = np.concatenate([rng.standard_normal((n, 2)) * rng.uniform(0.5, 2.0) + 0.1 for n in lengths])
    got = order.tree_sum(texel, terms, len(lengths))
    start = 0
    for k, n in enumerate(lengths):
        for ch in range(2):
            exact = np.float32(math.fsum(terms[start:start + n, ch]))
            assert abs(float(got[k, ch]) - float(exact)) <= float(np.spacing(abs(exact))), (n, ch, got[k, ch], exact)
        start += n
    # the tree is a function of the lengths: the same terms in a texel of their own give the same sum
    alone = order.tree_sum(np.zeros(lengths[-1], np.int64), terms[-lengths[-1]:], 1)
    assert np.array_equal(alone[0].view(np.int32), got[-1].view(np.int32))


def test_restated_terms_follow_the_corner_order():
    """On a 2 x 3 texture: one bilinear lookup based at (1, 2) gives texel (1, 2) its corner-00 term, (1, 0) its
    corner-01 term (column 2 + 1 wraps), (0, 2) corner 10 and (0, 0) corner 11; a lookup at an integer index has zero
    weights for three corners, which add +0.0."""
    idx = np.array([[1.25, 2.5], [0.0, 1.0]], np.float32)
    gout = np.array([[1.0], [2.0]], np.float32)
    texel, terms = order.ordered_terms(idx, gout, 1, 2, 3, 2, 'bilinear')
    w = {(1, 2): 0.75 * 0.5, (1, 0): 0.75 * 0.5, (0, 2): 0.25 * 0.5, (0, 0): 0.25 * 0.5}
    got = order.tree_sum(texel, terms, 6).reshape(2, 3)
    for (r, c), v in w.items():
        assert got[r, c] == np.float32(v), (r, c)
    assert got[0, 1] == 2.0 and got[1, 1] == 0.0 and not np.signbit(got).any()
