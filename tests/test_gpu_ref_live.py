"""GPU: the CUDA backward pass against the reference's own gradient kernel, run live.

oracle/_ref/libdirt_ref_grad.so is the reference's csrc/rasterise_grad_egl.cu compiled unmodified
(__graft_entry__.build() builds it wherever a reference checkout can be found, oracle/ref.py).  The stored fixtures of
test_ref_pin.py pin the CUDA path to it on small frames only; everything else was compared with the CPU oracle, this
project's own restatement of the kernel, which can share a misreading with the CUDA path.  Here every scene that
matters runs through both: the benched workloads at their benched sizes, every rare-path scene of test_gpu_paths.py
(kernel_paths.py), the four-slot variant build, a seeded sweep of random scenes, the backward flags and deferred
shading.

_check_live renders a scene with the library under test, takes its G-buffer from rasterise_visibility_raw (bit-exact
with the oracle, test_visibility_gbuffer_matches_oracle) and gives the reference kernel and the CUDA backward pass the
same pixels, G-buffer and seeded grad_pixels.  Bars are those of test_ref_pin.py: grad_background exact,
grad_vertices and grad_vertex_colors within rel_close (1e-4 relative), column 2 of grad_vertices exactly 0; the worst
ratios go into the end-of-run summary under names starting with 'ref-live:'.

The reference sums its vertex gradients with fp32 atomics in whatever order its threads run, so its output is not
reproducible to the bar on sums of tens of thousands of terms (two of its runs on the benched cube differ by more than
the bar in grad_vertex_colors).  It therefore runs with split = REF_SPLIT (oracle/ref.py assemble_grads): REF_SPLIT^2
runs, each with grad_pixels kept on one lattice of pixels (row and column modulo REF_SPLIT), summed in float64.  Every
per-pixel term and every dilation decision is still the reference kernel's own; each of its fp32 sums is 16 times
shorter.  Where the CPU oracle's backward pass is
affordable, its dilation decisions must also equal the reference kernel's, pixel for pixel and channel group by
channel group: one flipped pixel moves a vertex sum by far less than the gradient bar can see.

The library is only loaded here; these tests never read the reference checkout or build anything from it.
"""
import warnings

import numpy as np
import pytest

import kernel_paths as kp
from conftest import rel_close
import variant_builds
from test_gpu_paths import abi_backward, abi_forward

pytestmark = pytest.mark.gpu

# frames whose tiled framebuffer exceeds the H100's 2D surface limits (131072 x 65536) in the reference driver: the
# 65537-row frame of kp.RECORD_LIMIT_FRAMES.  They, and only they, are refused and skipped.
TOO_LARGE_FOR_REFERENCE = [(65537, 8)]   # (H, W)
ORACLE_MASK_IMAGES = 4                   # full frames of a large batch whose dilation masks the oracle checks
SWEEP_SCENES = 150
REF_SPLIT = 4                            # the reference's sums run over 4 x 4 pixel lattices (module docstring)
# Sweep scenes on which the CUDA path's own fp32 sums of strongly cancelling position terms (faces crossing w = 0) land
# further from the exact fp64 sum than this file's tensor-wide bar (seed 98: 1.87x from fp64, 2.4x from the reference's
# split sum on an H100): reported here, not asserted, because no fp32 summation order meets a 1e-4 bar relative to a
# sum that cancels.  test_gpu_det_records.py asserts every entry of that scene against the fp32 bound of its own terms
# (DESIGN.md section 2).
FP32_SUM_GAP = {98: ('grad_vertices',)}


@pytest.fixture(scope='module')
def ref(cuda_lib):
    from oracle import ref as r
    if not r.available():
        reason = ('oracle/_ref/libdirt_ref_grad.so is absent, so the CUDA backward pass was NOT compared with the '
                  'reference kernel: run __graft_entry__.build() where a reference checkout is found ($DIRT_REFERENCE, '
                  'or a `reference` directory beside the repository root) and bring oracle/_ref/ along to the GPU')
        warnings.warn(reason)   # also in the warnings summary of a run without -rs
        pytest.skip(reason)
    r.lib()
    return r


@pytest.fixture(scope='session')
def four_slot_lib(cuda_lib, tmp_path_factory):
    """The four-slot variant build of test_gpu_paths.py (variant_builds.py; compiled once per session)."""
    return variant_builds.four_slot_library(tmp_path_factory)


def _cuda(s):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.items()}


def _close(group, label, name, got, want, asserted=True):
    ok, ratio = rel_close(got, want, name='ref-live: %s %s%s' % (group, name, '' if asserted else ' (not asserted)'))
    assert ok or not asserted, '%s: %s off by %.2fx the tolerance from the reference kernel' % (label, name, ratio)


def _check_masks(oracle, s, pixels, gp, groups, ref_masks, label, images):
    """The oracle's dilation decisions against the reference kernel's, bit for bit, on the first `images` images.  The
    oracle also gets the next image, if there is one: a 1-wide group's flat-order taps at the end of an image read it."""
    n = min(images + 1, pixels.shape[0])
    _, _, _, masks = oracle.backward(s['vertices'][:n], s['faces'][:n], pixels[:n], gp[:n], groups, return_dilation=True)
    assert len(masks) == len(ref_masks)
    for g, (mo, mr) in enumerate(zip(masks, ref_masks)):
        mo, mr = mo[:images], mr[:images]
        bad = np.argwhere(mo != mr)
        assert bad.size == 0, '%s: channel group %d: the oracle dilates %d pixels the reference kernel does not and ' \
            'misses %d it does (first at [b, row, col] = %s)' % (label, g, int((mo & ~mr).sum()), int((mr & ~mo).sum()),
                                                                  bad[0].tolist())


def _check_live(L, ref, s, groups=None, label='', seed=0, group='', oracle=None, mask_images=None, flag_matrix=False,
                fp32_gap=()):
    """The CUDA backward pass of library L against the reference kernel on scene `s` (see the module docstring).
    The backward runs with the forward's face ids, with face ids re-derived inside the call and with the forward's
    workspace reused; with flag_matrix also SHARED_GEOMETRY and each SKIP_* flag.  With `oracle`, the dilation masks of
    the first `mask_images` images (all if None) are compared as well.  `fp32_gap` names outputs measured but not
    asserted (see FP32_SUM_GAP).  Returns the reference's dilation masks.
    Raises ref.FrameTooLarge, before any CUDA backward runs, for a frame the reference driver cannot hold."""
    import torch
    from dirt_b200 import rasterise_ops as ops
    t = _cuda(s)
    B, H, W, C = s['background'].shape
    V = s['vertices'].shape[1]
    pixels = torch.empty_like(t['background'])
    ids = torch.empty((B, H, W), dtype=torch.int32, device='cuda')
    ws = abi_forward(L, t['background'], t['vertices'], t['vertex_colors'], t['faces'], pixels, ids)
    vis_ids, gbuf = ops.rasterise_visibility_raw(t['vertices'], t['faces'], H, W)
    assert torch.equal(vis_ids, ids), label + ': the visibility pass and the forward pass disagree on face ids'
    px_np, ids_np, gbuf_np = pixels.cpu().numpy(), ids.cpu().numpy(), gbuf.cpu().numpy()
    del vis_ids, gbuf
    gp_np = np.random.default_rng(seed).standard_normal(px_np.shape).astype(np.float32)
    gb_r, gv_r, gc_r, masks_r = ref.backward(s['vertices'], s['faces'], px_np, gp_np, gbuf_np, ids_np, groups,
                                             return_dilation=True, split=REF_SPLIT)
    del gbuf_np
    assert (gv_r[..., 2] == 0).all()
    if oracle is not None:
        _check_masks(oracle, s, px_np, gp_np, groups, masks_r, label, B if mask_images is None else mask_images)
    gp = torch.from_numpy(gp_np).cuda()

    def close(lab, name, got, want):
        _close(group, lab, name, got, want, asserted=name not in fp32_gap)

    def run(face_ids, flags=0, reuse=False):
        lead = () if flags & 1 else (B,)
        gb, gv, gc = torch.empty_like(pixels), torch.empty(lead + (V, 4), device='cuda'), torch.empty(lead + (V, C), device='cuda')
        abi_backward(L, t['vertices'], t['faces'], pixels, gp, face_ids, gb, gv, gc, groups, flags, ws if reuse else None,
                     reuse)
        return gb.cpu().numpy(), gv.cpu().numpy(), gc.cpu().numpy()

    for how, face_ids, reuse in (('ids passed', ids, False), ('ids re-derived', None, False), ('workspace reused', ids, True)):
        gb, gv, gc = run(face_ids, reuse=reuse)
        lab = '%s (%s)' % (label, how)
        assert np.array_equal(gb, gb_r), lab + ': grad_background differs from the reference kernel'
        close(lab, 'grad_vertices', gv, gv_r)
        close(lab, 'grad_vertex_colors', gc, gc_r)
        assert (gv[..., 2] == 0).all(), lab + ': grad_vertices[..., 2] is not 0'
    if flag_matrix:
        _, gv, gc = run(ids, flags=1)   # DIRT_BWD_SHARED_GEOMETRY: sums over the batch
        close(label + ' (shared geometry)', 'grad_vertices', gv, gv_r.astype(np.float64).sum(0))
        close(label + ' (shared geometry)', 'grad_vertex_colors', gc, gc_r.astype(np.float64).sum(0))
        gb, gv, gc = run(ids, flags=2)  # DIRT_BWD_SKIP_POSITION
        assert np.array_equal(gb, gb_r), label + ' (skip position): grad_background differs'
        close(label + ' (skip position)', 'grad_vertex_colors', gc, gc_r)
        assert not gv.any()
        _, gv, gc = run(ids, flags=4)   # DIRT_BWD_SKIP_COLOUR
        close(label + ' (skip colour)', 'grad_vertices', gv, gv_r)
        assert not gc.any()
    return masks_r


# ---- 1. the benched workloads at their benched sizes -------------------------------------------------------------------

def _bench_workloads():
    import bench
    return [(name,) + bench.WORKLOADS[name][:2] for name in sorted(bench.WORKLOADS)]


@pytest.mark.parametrize('name,gen,kwargs', _bench_workloads(), ids=[w[0] for w in _bench_workloads()])
def test_benched_workload(cuda_lib, ref, oracle, name, gen, kwargs):
    """cfg3 (B = 64, 512^2, C = 4: the fused {3,1} launch), cfg4 (B = 32, C = 3), cfg5 (B = 64, 1024^2, 49 728 faces),
    cube (B = 64, 640 x 480, 12 faces: flat-shaded silhouettes full of near-tie dilation decisions) and cfg2, as
    bench.py renders them; the backward flags on cfg3 and cfg4; dilation masks of the first four images."""
    from dirt_b200 import scenes
    s = getattr(scenes, gen)(**kwargs)
    masks = _check_live(cuda_lib, ref, s, None, 'bench %s' % name, seed=17, group='bench', oracle=oracle,
                        mask_images=None if name in ('cube', 'cfg2') else ORACLE_MASK_IMAGES,
                        flag_matrix=name in ('cfg3', 'cfg4'))
    assert all(m.any() for m in masks), 'bench %s: no pixel dilated, the mask comparison saw nothing' % name


# ---- 2. the rare-path scenes of test_gpu_paths.py ----------------------------------------------------------------------

@pytest.mark.parametrize('W', kp.OVERFLOW_WIDTHS)
@pytest.mark.parametrize('channels,groups', kp.OVERFLOW_CHANNELS)
def test_face_table_overflow(cuda_lib, ref, oracle, channels, groups, W):
    _check_live(cuda_lib, ref, kp.overflow_scene(channels, W), groups, 'overflow C=%d groups=%s W=%d' % (channels, groups, W),
                group='paths', oracle=oracle)


@pytest.mark.parametrize('W', kp.OVERFLOW_WIDTHS)
@pytest.mark.parametrize('channels,groups', kp.OVERFLOW_CHANNELS)
def test_exactly_full_face_table(cuda_lib, ref, oracle, channels, groups, W):
    _check_live(cuda_lib, ref, kp.full_table_scene(channels, W), groups, 'full table C=%d groups=%s W=%d' % (channels, groups, W),
                group='paths', oracle=oracle)


@pytest.mark.parametrize('W', kp.FLAT_ORDER_WIDTHS)
@pytest.mark.parametrize('channels,groups', kp.FLAT_ORDER_CHANNELS)
def test_flat_order_reads_across_images(cuda_lib, ref, oracle, channels, groups, W):
    """1-wide groups read "channels" 1 and 2 of a pixel from the next two pixels in flat order; at the end of an image
    those are the next image's first pixels, and every pixel of these frames is covered."""
    _check_live(cuda_lib, ref, kp.flat_order_scene(channels, W, seed=W), groups,
                'flat order C=%d groups=%s W=%d' % (channels, groups, W), seed=W, group='paths', oracle=oracle)


def test_batch_past_the_grid_limit(cuda_lib, ref, oracle):
    s = kp.grid_limit_scene()
    _check_live(cuda_lib, ref, s, None, 'grid limit B=%d' % s['background'].shape[0], seed=1, group='paths', oracle=oracle)


@pytest.mark.parametrize('channels', kp.RECORD_LIMIT_CHANNELS)
@pytest.mark.parametrize('H,W', kp.RECORD_LIMIT_FRAMES)
def test_shading_record_limit(cuda_lib, ref, oracle, H, W, channels):
    s = kp.edge_strip(H, W, channels, seed=channels)
    label = 'record limit %dx%d C=%d' % (W, H, channels)
    if (H, W) in TOO_LARGE_FOR_REFERENCE:
        with pytest.raises(ref.FrameTooLarge):
            _check_live(cuda_lib, ref, s, None, label, group='paths')
        pytest.skip('%s: %d rows exceed the 2D surface height the reference driver binds its G-buffer to' % (label, H))
    _check_live(cuda_lib, ref, s, None, label, group='paths', oracle=oracle)


@pytest.mark.parametrize('batch', [1, 2])
def test_depth_ties(cuda_lib, ref, oracle, batch):
    _check_live(cuda_lib, ref, kp.coplanar_tie_scene(batch=batch), None, 'ties B=%d' % batch, group='paths', oracle=oracle)


# ---- 3. every tile through tile_generic: the four-slot variant build ---------------------------------------------------

@pytest.mark.parametrize('channels,groups', kp.OVERFLOW_CHANNELS)
def test_four_slot_overflow(four_slot_lib, ref, oracle, channels, groups):
    for W in kp.OVERFLOW_WIDTHS:
        _check_live(four_slot_lib, ref, kp.overflow_scene(channels, W), groups,
                    'slots=4 overflow C=%d groups=%s W=%d' % (channels, groups, W), group='four-slot',
                    oracle=oracle, flag_matrix=channels == 4)


@pytest.mark.parametrize('channels,groups', kp.FLAT_ORDER_CHANNELS)
def test_four_slot_flat_order(four_slot_lib, ref, oracle, channels, groups):
    for W in kp.FLAT_ORDER_WIDTHS:
        _check_live(four_slot_lib, ref, kp.flat_order_scene(channels, W, seed=W), groups,
                    'slots=4 flat order C=%d groups=%s W=%d' % (channels, groups, W), seed=W, group='four-slot',
                    oracle=oracle)


@pytest.mark.parametrize('seed', [0, 1, 2])
@pytest.mark.parametrize('channels', [1, 3, 4, 5])
def test_four_slot_soup(four_slot_lib, ref, oracle, seed, channels):
    from dirt_b200 import scenes
    s = scenes.random_soup(batch=2, width=61, height=45, n_faces=70, channels=channels, seed=seed)
    _check_live(four_slot_lib, ref, s, None, 'slots=4 soup C=%d seed=%d' % (channels, seed), seed=seed, group='four-slot',
                oracle=oracle)


# ---- 4. a seeded sweep of random scenes --------------------------------------------------------------------------------

def random_groups(rng, C):
    """A random valid grouping of C channels into widths 1 and 3."""
    groups, left = [], C
    while left:
        groups.append(3 if left >= 3 and rng.random() < 0.6 else 1)
        left -= groups[-1]
    return groups


def sweep_scene(seed):
    """One random scene: B 1-6, H and W 1-96 (some frames have no interior pixel), C 1-8 with a random grouping, a
    soup of shared vertices with some behind the camera (w <= 0) and some past the guard band, degenerate faces
    (a repeated vertex), out-of-range indices, duplicated faces (another face's vertex triple) and, in every third
    scene, a NaN vertex."""
    rng = np.random.default_rng(1000 + seed)
    B, H, W, C = int(rng.integers(1, 7)), int(rng.integers(1, 97)), int(rng.integers(1, 97)), int(rng.integers(1, 9))
    F = int(rng.integers(1, 90))
    V = int(rng.integers(3, F + 12))
    w = rng.uniform(0.4, 3.0, (B, V))
    w = np.where(rng.random((B, V)) < 0.1, -rng.uniform(0.05, 1.0, (B, V)), w)
    xy = rng.uniform(-1.4, 1.4, (B, V, 2)) * np.abs(w)[..., None]
    xy = np.where(rng.random((B, V, 1)) < 0.04, xy * 1e6, xy)
    z = rng.uniform(-1.2, 1.2, (B, V)) * np.abs(w)
    vertices = np.concatenate([xy, z[..., None], w[..., None]], axis=2).astype(np.float32)
    faces = rng.integers(0, V, (B, F, 3)).astype(np.int32)
    pick = rng.random((B, F))
    faces[..., 1] = np.where(pick < 0.05, faces[..., 0], faces[..., 1])                          # degenerate
    faces[..., 2] = np.where((pick >= 0.05) & (pick < 0.08), V + rng.integers(0, 3, (B, F)), faces[..., 2])
    faces[..., 0] = np.where((pick >= 0.08) & (pick < 0.10), -1, faces[..., 0])                   # out of range
    src = rng.integers(0, F, (B, F))
    dup = (pick >= 0.10) & (pick < 0.15)
    faces = np.where(dup[..., None], np.take_along_axis(faces, np.repeat(src[..., None], 3, 2), 1), faces)
    if seed % 3 == 0:
        vertices[int(rng.integers(0, B)), int(rng.integers(0, V)), int(rng.integers(0, 4))] = np.nan
    s = dict(background=rng.uniform(size=(B, H, W, C)).astype(np.float32), vertices=vertices,
             vertex_colors=rng.uniform(-1.0, 1.0, (B, V, C)).astype(np.float32), faces=faces.astype(np.int32))
    return s, random_groups(rng, C)


@pytest.mark.parametrize('seed', range(SWEEP_SCENES))
def test_random_scene(cuda_lib, ref, oracle, seed):
    s, groups = sweep_scene(seed)
    B, H, W, C = s['background'].shape
    _check_live(cuda_lib, ref, s, groups, 'sweep seed=%d (B=%d %dx%d C=%d groups=%s)' % (seed, B, W, H, C, groups),
                seed=seed, group='sweep', oracle=oracle, fp32_gap=FP32_SUM_GAP.get(seed, ()))


# ---- 5. deferred shading -----------------------------------------------------------------------------------------------

def _deferred_scene(name):
    from dirt_b200 import scenes
    if name == 'small':
        return scenes.bent_square_scene(channels=7, seed=5)
    s = scenes.config3(batch=8, width=512, height=512, background='uniform')
    rng = np.random.default_rng(9)
    B, H, W, _ = s['background'].shape
    V = s['vertices'].shape[1]
    s['vertex_colors'] = np.concatenate([s['vertex_colors'], rng.uniform(-1, 1, (B, V, 3)).astype(np.float32)], -1)
    s['background'] = rng.uniform(size=(B, H, W, 7)).astype(np.float32)
    return s


@pytest.mark.parametrize('name', ['small', 'cfg3'])
def test_deferred_matches_reference_recipe(cuda_lib, ref, name):
    """rasterise_batch_deferred with a nonlinear shader against the reference's recipe (dirt/rasterise_ops.py:180-257)
    evaluated with the reference kernel: the vertex gradient is its backward pass on the SHADED pixels, the attribute and
    background gradients its backward pass on the G-buffer with the shader's d_gbuffer from torch autograd."""
    import torch
    import dirt_b200 as dirt
    from dirt_b200 import rasterise_ops as ops
    s = _deferred_scene(name)
    t = _cuda(s)
    B, H, W, _ = s['background'].shape
    for k in ('background', 'vertices', 'vertex_colors'):
        t[k].requires_grad_(True)
    light = torch.tensor([0.3, 0.5, 0.8], device='cuda', requires_grad=True)

    def shader_fn(gbuffer, light):
        return gbuffer[..., :3] * (gbuffer[..., 3:6] * light).sum(-1, keepdim=True).abs() + 0.1 * gbuffer[..., 6:]

    pixels = dirt.rasterise_batch_deferred(t['background'], t['vertices'], t['vertex_colors'], t['faces'], shader_fn, [light])
    gp = torch.from_numpy(np.random.default_rng(0).standard_normal(tuple(pixels.shape)).astype(np.float32)).cuda()
    (pixels * gp).sum().backward()

    attrs, ids = ops.rasterise_forward_raw(t['background'].detach(), t['vertices'].detach(), t['vertex_colors'].detach(),
                                           t['faces'])
    vis_ids, gbuf = ops.rasterise_visibility_raw(t['vertices'].detach(), t['faces'], H, W)
    assert torch.equal(vis_ids, ids)
    g = attrs.clone().requires_grad_(True)
    d_gbuf, = torch.autograd.grad(shader_fn(g, light.detach()), [g], gp)
    args = (s['vertices'], s['faces'])
    _, gv_r, _ = ref.backward(*args, pixels.detach().cpu().numpy(), gp.cpu().numpy(), gbuf.cpu().numpy(), ids.cpu().numpy(),
                              split=REF_SPLIT)
    gb_r, _, gc_r = ref.backward(*args, attrs.cpu().numpy(), d_gbuf.cpu().numpy(), gbuf.cpu().numpy(), ids.cpu().numpy(),
                                 split=REF_SPLIT)
    label = 'deferred %s' % name
    _close('deferred', label, 'grad_vertices', t['vertices'].grad.cpu().numpy(), gv_r)
    _close('deferred', label, 'grad_vertex_colors', t['vertex_colors'].grad.cpu().numpy(), gc_r)
    assert np.array_equal(t['background'].grad.cpu().numpy(), gb_r), label + ': grad_background differs'
