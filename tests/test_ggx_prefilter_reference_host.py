"""CPU: tests/ggx_prefilter_reference.py against the dense restatement it slices, at the sizes the dense one reaches."""
import numpy as np
import pytest
import torch

import cubemap_ggx_restatement as ibl
import cubemap_restatement as cm
import ggx_prefilter_reference as ref


@pytest.mark.parametrize('S', [16, 32, 48, 64])
def test_rows_and_columns_are_the_dense_weights(S):
    rng = np.random.default_rng(S)
    L = ibl.level_count(S)
    for k in range(1, L):
        dense, s = ibl.weights(k, L, S)
        assert ref.level_source(k, S)[0] == s
        n_out, n_src = dense.shape
        idx = np.unique(np.concatenate([[0, n_out - 1], rng.integers(0, n_out, min(n_out, 200))]))
        w, W = ref.rows(k, S, idx)
        want = dense[idx]
        got = w.toarray()
        assert w.nnz == np.count_nonzero(got) and np.array_equal(got > 0, want > 0), (S, k)
        assert np.abs(got - want).max() <= 1e-15 * np.abs(want).max(), (S, k)
        assert np.allclose(W, want.sum(1), rtol=1e-14, atol=0), (S, k)
        jdx = np.unique(np.concatenate([[0, n_src - 1], rng.integers(0, n_src, min(n_src, 200))]))
        col = ref.columns(k, S, jdx)
        got, want = col.toarray(), dense[:, jdx].T
        assert col.nnz == np.count_nonzero(got) and np.array_equal(got > 0, want > 0), (S, k)
        assert np.abs(got - want).max() <= 1e-15 * np.abs(want).max(), (S, k)


@pytest.mark.parametrize('S', [16, 32, 48, 64])
def test_the_float64_predecision_agrees_with_the_fp32_support(S):
    """Every pair the float64 cosine decides, over all pairs of every level, is decided the same way by the fp32 one;
    the band it leaves to the fp32 test is a small share of the pairs."""
    L = ibl.level_count(S)
    undecided_total = pairs = 0
    for k in range(1, L):
        s, _, ck = ref.level_source(k, S)
        rd = ibl.texel_table(S >> k)[0].reshape(-1, 3)
        ld = ibl.texel_table(S >> s)[0].reshape(-1, 3)
        _, exact = ibl.support(rd, ld, ck)
        inside, undecided = ref.decide(rd.astype(np.float64) @ ld.astype(np.float64).T, ck)
        assert not (inside & ~exact).any() and not (~inside & ~undecided & exact).any(), (S, k)
        undecided_total += int(undecided.sum())
        pairs += undecided.size
    assert undecided_total < 0.01 * pairs


def test_adjoint_rows_is_the_transposed_dense_prefilter():
    S, C = 32, 2
    rng = np.random.default_rng(1)
    L, ss = ibl.level_count(S), ibl.source_cap(S)
    grads = {k: rng.standard_normal((6 * (S >> k) ** 2, C)) for k in range(1, L)}
    W = {k: ibl.weights(k, L, S)[0].sum(1) * (1 + 1e-3 * rng.random(6 * (S >> k) ** 2)) for k in range(1, L)}
    for s in range(1, ss + 1):
        jdx = rng.integers(0, 6 * (S >> s) ** 2, 50)
        want = sum(ibl.weights(k, L, S)[0].T @ (grads[k] / W[k][:, None])
                   for k in range(1, L) if min(k, ss) == s)[jdx]
        assert np.allclose(ref.adjoint_rows(S, s, jdx, grads, W), want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


@pytest.mark.parametrize('Sk', [1, 2, 3, 7, 15, 16, 30, 60, 64, 120, 240])
def test_exact_centre_directions_land_on_integer_padded_coordinates(Sk):
    n = 6 * Sk * Sk
    ok = ref.has_exact_centre(0, Sk, np.arange(n))
    # every texel of a power-of-two edge; elsewhere all but a few low indices (see _edge_centres)
    assert ok.all() if Sk & (Sk - 1) == 0 else ok.mean() > 0.65
    d = torch.from_numpy(ref.exact_centre_directions(0, Sk, np.arange(n)))
    assert torch.isnan(d).any(-1).numpy().tolist() == (~ok).tolist()
    face, s, t, valid = cm.face_coords(d[ok])
    pr, pc = (t * Sk - 0.5) + 1., (s * Sk - 0.5) + 1.
    f, rc = np.divmod(np.arange(n)[ok], Sk * Sk)
    assert valid.all() and np.array_equal(face.numpy(), f)
    assert np.array_equal(pr.numpy(), rc // Sk + 1.) and np.array_equal(pc.numpy(), rc % Sk + 1.)
    # at a level k of a larger map the same texel grid
    assert np.array_equal(ref.exact_centre_directions(2, 4 * Sk, np.arange(n)), d.numpy(), equal_nan=True)
