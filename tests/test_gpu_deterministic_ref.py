"""GPU: the deterministic backward pass against the reference's own gradient kernel, run live (oracle/_ref, see
test_gpu_ref_live.py for how the reference runs and why its sums are split over 4 x 4 pixel lattices).

The scenes are the benched workloads at their benched sizes and the 150 scenes of the seeded sweep, with no exception:
random scene 98, whose faces cross w = 0 and whose cancelling position terms put the default path's fp32 sums of
grad_vertices past the bar, is asserted here, because this path sums in float64.  Bars are those of test_gpu_ref_live.py:
grad_background exact, grad_vertices and grad_vertex_colors within rel_close, column 2 exactly 0; the dilation codes must
mark exactly the pixels the reference kernel dilates.  The worst ratios go into the end-of-run summary under names
starting with 'ref-live deterministic:'.  Without oracle/_ref the file skips with a warning."""
import numpy as np
import pytest

from conftest import rel_close
from test_gpu_deterministic import codes, det_call
from test_gpu_ref_live import REF_SPLIT, SWEEP_SCENES, ref, sweep_scene   # noqa: F401 (ref is a fixture)

pytestmark = pytest.mark.gpu

SCENE_98 = 98   # the sweep scene of test_gpu_ref_live.FP32_SUM_GAP


def _cuda(s):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.items()}


def check_live(ref, s, groups, label, group, seed=0):
    import torch
    from dirt_b200 import rasterise_ops as ops
    t = _cuda(s)
    B, H, W, C = s['background'].shape
    pixels, ids = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    vis_ids, gbuf = ops.rasterise_visibility_raw(t['vertices'], t['faces'], H, W)
    assert torch.equal(vis_ids, ids), label + ': the visibility pass and the forward pass disagree on face ids'
    px_np, ids_np = pixels.cpu().numpy(), ids.cpu().numpy()
    gp_np = np.random.default_rng(seed).standard_normal(px_np.shape).astype(np.float32)
    gb_r, gv_r, gc_r, masks_r = ref.backward(s['vertices'], s['faces'], px_np, gp_np, gbuf.cpu().numpy(), ids_np, groups,
                                             return_dilation=True, split=REF_SPLIT)
    del gbuf, vis_ids
    gb, gv, gc, scratch = det_call(t, pixels, torch.from_numpy(gp_np).cuda(), ids, groups)
    assert np.array_equal(gb.cpu().numpy(), gb_r), label + ': grad_background differs from the reference kernel'
    ratios = {}
    for name, got, want in (('grad_vertices', gv, gv_r), ('grad_vertex_colors', gc, gc_r)):
        ok, ratios[name] = rel_close(got.cpu().numpy(), want, name='ref-live deterministic: %s %s' % (group, name))
        assert ok, '%s: %s off by %.2fx the tolerance from the reference kernel' % (label, name, ratios[name])
    assert (gv[..., 2] == 0).all()
    cp = codes(scratch, B, H, W, len(masks_r))
    for g, m in enumerate(masks_r):
        np.testing.assert_array_equal((cp[g] & 3) >= 2, np.asarray(m, bool), err_msg=label + ': dilation of group %d' % g)
    return ratios


def _bench_workloads():
    import bench
    return [(name,) + bench.WORKLOADS[name][:2] for name in sorted(bench.WORKLOADS)]


@pytest.mark.parametrize('name,gen,kwargs', _bench_workloads(), ids=[w[0] for w in _bench_workloads()])
def test_benched_workload(cuda_lib, ref, name, gen, kwargs):
    from dirt_b200 import scenes
    check_live(ref, getattr(scenes, gen)(**kwargs), None, 'bench %s' % name, 'bench', seed=17)


@pytest.mark.parametrize('seed', range(SWEEP_SCENES))
def test_random_scene(cuda_lib, ref, seed):
    s, groups = sweep_scene(seed)
    B, H, W, C = s['background'].shape
    ratios = check_live(ref, s, groups, 'sweep seed=%d (B=%d %dx%d C=%d groups=%s)' % (seed, B, W, H, C, groups), 'sweep',
                        seed=seed)
    if seed == SCENE_98:
        print('sweep scene 98: grad_vertices at %.3fx the bar from the reference kernel' % ratios['grad_vertices'])
