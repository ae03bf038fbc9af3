"""GPU: the triangle-setup kernel's own timer, and its two vertex-colour gathers (one 16-byte row per vertex for C = 4 with
16-byte aligned colours, scalar loads otherwise) against each other and against the CPU oracle, on batches whose faces do
not fill whole warps, so that one warp holds faces of two images and the last warp is partly empty."""
import numpy as np
import pytest

from conftest import rel_close
from dirt_b200 import scenes

pytestmark = pytest.mark.gpu


def test_setup_kernel_timer(cuda_lib):
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=2, width=64, height=64, level=1)
    t = {k: torch.from_numpy(v).cuda() for k, v in s.items()}
    assert cuda_lib.dirt_kernel_timer_enable(3) == 0
    pixels, ids = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'])
    ms = float(cuda_lib.dirt_kernel_timer_elapsed_ms())
    assert 0.0 < ms < 1000.0
    # a backward call without the forward's workspace runs the setup kernel again (records only, no binning)
    assert cuda_lib.dirt_kernel_timer_enable(3) == 0
    ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, torch.ones_like(pixels), ids)
    assert 0.0 < float(cuda_lib.dirt_kernel_timer_elapsed_ms()) < 1000.0
    assert cuda_lib.dirt_kernel_timer_enable(0) == 0


@pytest.mark.parametrize('level,batch', [(1, 3), (2, 5)])   # F = 80 and 320: B*F = 240 and 1600
def test_colour_rows_aligned_and_unaligned(cuda_lib, oracle, level, batch):
    import torch
    from dirt_b200 import rasterise_ops as ops
    s = scenes.config3(batch=batch, width=96, height=80, level=level, background='uniform')
    t = {k: torch.from_numpy(v).cuda() for k, v in s.items()}
    colours = t['vertex_colors']
    assert colours.data_ptr() % 16 == 0
    flat = torch.empty(colours.numel() + 1, dtype=torch.float32, device='cuda')
    shifted = flat[1:].view(colours.shape)   # 4-byte aligned, not 16: the scalar gathers
    shifted.copy_(colours)
    assert shifted.data_ptr() % 16 != 0
    out = [ops.rasterise_forward_raw(t['background'], t['vertices'], c, t['faces']) for c in (colours, shifted)]
    (p_a, ids_a), (p_b, ids_b) = [(p.cpu().numpy(), i.cpu().numpy()) for p, i in out]
    np.testing.assert_array_equal(ids_a, ids_b)
    np.testing.assert_array_equal(p_a.view(np.int32), p_b.view(np.int32))
    pixels_o, ids_o = oracle.forward(**s, return_face_ids=True)
    np.testing.assert_array_equal(ids_a, ids_o)
    ok, ratio = rel_close(p_a, pixels_o, name='pixels vs oracle')
    assert ok, 'pixels off by %.2fx the tolerance' % ratio
