"""The grids of the kernels that cap their grid and loop past the cap, restated in Python, and the sizes of the scenes
tests/test_gpu_launch_limits.py runs to take those loops past their first round.

CPU only.  Each function restates the launch arithmetic of one place in dirt_b200/csrc, named in its docstring; `caps` is
a dict of the compile-time caps (SHIPPED, or variant_builds.SMALL_GRID_CAPS).  tests/test_launch_limits.py shows that
every scene crosses the boundary it is there for, by at least one full round and a partial one.
"""
from variant_builds import SMALL_GRID_CAPS

SHIPPED = {'DIRT_TEX_MAX_BLOCKS': 1 << 16, 'DIRT_TEX_DET_GRID': 8192, 'DIRT_LIGHT_MAX_ITEMS_PER_GRID': 65535,
           'DIRT_LIGHT_REDUCE_MAX_BLOCKS': 1 << 20, 'DIRT_NORMALS_MAX_BLOCKS': 1 << 20, 'DIRT_DET_MAX_BLOCKS': 1 << 20,
           'DIRT_DERIV_MAX_BLOCKS': 0x7fffffff}
SMALL = SMALL_GRID_CAPS

TEX_THREADS = 256       # texture.cu TEX_THREADS
RS_TILE = 4096          # texture.cu RS_TILE: lookups per sort tile
RS_THREADS = 256        # texture.cu RS_THREADS: tiles per round of tex_sort_scan_kernel
DET_CHUNK = 4096        # texture.cu DET_CHUNK: terms per chunk of a texel's sum
DET_WARPS = 8           # TEX_THREADS / 32: texels (gather) or chunk slots (chunk kernel) per CTA and round
LIGHT_THREADS = 256     # common.cuh LIGHT_THREADS: points per chunk
NORMALS_THREADS = 256   # common.cuh NORMALS_THREADS
DET_THREADS = 256       # deterministic.cu DET_THREADS
DERIV_THREADS = 256     # derivatives.cu DERIV_THREADS


def rounds(work, stride):
    """Rounds of a grid-stride loop over `work` items that advances by `stride` items a round."""
    return -(-work // stride)


def crosses(work, stride):
    """The loop runs one full round and then at least a partial one, the last round partial."""
    return work > stride and work % stride != 0


def tex_blocks(work, caps):
    """texture.cu blocks_for: ceil(work / TEX_THREADS) CTAs, at most DIRT_TEX_MAX_BLOCKS."""
    return min(-(-work // TEX_THREADS), caps['DIRT_TEX_MAX_BLOCKS'])


def tex_forward(total, C, caps):
    """(work, stride) of the forward lookup (texture.cu forward_ct): one thread per lookup for C in 1..4 and for the
    trilinear lookup, else texture_forward_generic_kernel, one thread per output element."""
    work = total if 1 <= C <= 4 else total * C
    return work, tex_blocks(work, caps) * TEX_THREADS


def generic_step(total, C, caps):
    """(step_g, step_c) of texture_forward_generic_kernel (texture.cu forward_ct): the stride in elements split into whole
    lookups and the channels left over; step_c != 0 makes the loop wrap the channel."""
    step = tex_blocks(total * C, caps) * TEX_THREADS
    return step // C, step % C


def sort_tiles(total):
    """Sort tiles of the deterministic texture backward (texture.cu launch_texture_backward_deterministic)."""
    return -(-total // RS_TILE)


def scan_rounds(total):
    """Rounds of tex_sort_scan_kernel's loop over the tiles, each carrying the sum of the ones before."""
    return rounds(sort_tiles(total), RS_THREADS)


def sort_passes(sentinel):
    """texture.cu sort_passes: one 8-bit pass per byte of the sentinel TB * TH * TW."""
    return (sentinel.bit_length() + 7) // 8


def det_blocks(work, per_block, caps):
    """texture.cu det_blocks: ceil(work / per_block) CTAs, at least 1, at most DIRT_TEX_DET_GRID."""
    return max(1, min(-(-work // per_block), caps['DIRT_TEX_DET_GRID']))


def segment_bounds(texels, caps):
    """(work, stride) of tex_segment_bounds_kernel: one thread per key 0 .. sentinel + 1."""
    work = texels + 2
    return work, det_blocks(work, TEX_THREADS, caps) * TEX_THREADS


def gather(texels, caps):
    """(work, stride) of tex_det_gather_kernel: one warp per texel."""
    return texels, det_blocks(texels, DET_WARPS, caps) * DET_WARPS


def chunk_slots(terms_per_texel):
    """Chunk slots the gather kernel hands out: ceil(L / DET_CHUNK) for every texel of more than DET_CHUNK terms."""
    return sum(-(-L // DET_CHUNK) for L in terms_per_texel if L > DET_CHUNK)


def chunk(total, mode, slots, caps):
    """(work, stride) of tex_det_chunk_kernel: one warp per slot, over a grid sized for twice the slots of the terms."""
    terms = total * (4 if mode == 'bilinear' else 1)
    return slots, det_blocks(2 * -(-terms // DET_CHUNK), DET_WARPS, caps) * DET_WARPS


def finish(total, mode, listed, C, caps):
    """(work, stride) of tex_det_finish_kernel: one thread per (listed texel, channel)."""
    terms = total * (4 if mode == 'bilinear' else 1)
    return listed * C, det_blocks((terms // (DET_CHUNK + 1) + 1) * C, TEX_THREADS, caps) * TEX_THREADS


def mip_build(TB, TH, TW, C, k, caps):
    """(work, stride) of mip_build_kernel making level k: one thread per element of the level."""
    work = TB * (TH >> k) * (TW >> k) * C
    return work, tex_blocks(work, caps) * TEX_THREADS


def mip_collapse(TB, TH, TW, C, caps):
    """(work, stride) of mip_collapse_kernel: one thread per element of level 0."""
    work = TB * TH * TW * C
    return work, tex_blocks(work, caps) * TEX_THREADS


def point_grid(B, caps):
    """(work, stride) of the item loop of the lighting, GGX and SH kernels (lighting.cu point_grid / sh_grid): gridDim.y
    = min(B, DIRT_LIGHT_MAX_ITEMS_PER_GRID)."""
    return B, min(B, caps['DIRT_LIGHT_MAX_ITEMS_PER_GRID'])


def reduce_grid(total, caps):
    """(work, stride) of lighting_reduce_kernel (lighting.cu reduce_params and launch_sh_lighting_backward): one CTA per
    output element, at most DIRT_LIGHT_REDUCE_MAX_BLOCKS."""
    return total, min(total, caps['DIRT_LIGHT_REDUCE_MAX_BLOCKS'])


def param_columns(model, C):
    """Columns of the parameter gradients of one item (lighting.cu param_jobs; SH: the 9 x C coefficients)."""
    return {'diffuse_directional': 3 + C, 'diffuse_point': 3 + C, 'specular_directional': 3 + C + 3 + 1,
            'ggx': 3 + C + 3, 'ggx_point': 3 + C + 3, 'sh': 9 * C}[model]


def normals_blocks(work, caps):
    """normals.cu blocks_for: ceil(work / NORMALS_THREADS) CTAs, at least 1, at most DIRT_NORMALS_MAX_BLOCKS."""
    return max(1, min(-(-work // NORMALS_THREADS), caps['DIRT_NORMALS_MAX_BLOCKS']))


def normals_loops(items, V, F, caps):
    """(work, stride) of the normals kernels: count / fill over the F faces, rank over the 3F corners (normals.cu
    launch_corner_adjacency), forward and backward over the items * V rows."""
    return {name: (n, normals_blocks(n, caps) * NORMALS_THREADS)
            for name, n in (('faces', F), ('corners', 3 * F), ('rows', items * V))}


def det_raster_loops(B, H, W, V, F, caps):
    """(work, stride) of the deterministic rasteriser backward (deterministic.cu det_blocks): det_record_kernel over
    the pixels, det_face_warp_kernel over the faces (one warp each), det_vertex_kernel over the B * V rows."""
    def blocks(n, per_block):
        return max(1, min(-(-n // per_block), caps['DIRT_DET_MAX_BLOCKS']))
    px, faces, rows = B * H * W, B * F, B * V
    return {'pixels': (px, blocks(px, DET_THREADS) * DET_THREADS),
            'faces': (faces, blocks(faces, DET_THREADS // 32) * (DET_THREADS // 32)),
            'rows': (rows, blocks(rows, DET_THREADS) * DET_THREADS)}


def derivatives_loop(B, H, W, caps):
    """(work, stride) of derivatives_kernel: one thread per pixel, at most DIRT_DERIV_MAX_BLOCKS CTAs."""
    px = B * H * W
    return px, min(-(-px // DERIV_THREADS), caps['DIRT_DERIV_MAX_BLOCKS']) * DERIV_THREADS


# ---- the scenes of tests/test_gpu_launch_limits.py -------------------------------------------------------------------

# (a) the small-grid variant against the product
VAR_TEX_SHAPE = (37, 29)           # texture of the lookups, one image
VAR_TEX_LOOKUPS = 3001             # before the 78 edge lookups of test_gpu_texture._indices
VAR_TEX_CHANNELS = [1, 2, 3, 4, 5, 6, 7, 8]
VAR_DET_LONG = (13, 11)            # texture of det_long_indices: every texel gets more than DET_CHUNK terms
VAR_DET_LONG_CHANNELS = [4, 5]
VAR_MIP_SHAPE = (2, 46, 42)        # TB, TH, TW of the trilinear lookups: levels 46x42 and 23x21
VAR_LIGHT_B, VAR_LIGHT_V = 11, 333
VAR_LIGHT_CHANNELS = [3, 5]
VAR_NORMALS_ITEMS = 3
VAR_NORMALS_FAN = 5000             # faces of the fan mesh
VAR_OVERFLOW_W = 62                # width of kernel_paths.overflow_scene
VAR_SOUP = dict(batch=2, width=61, height=45, n_faces=450, seed=3)
VAR_DERIV_SOUP = dict(batch=4, width=80, height=56, n_faces=50, channels=6, seed=5, behind_camera=True)



def det_long_indices():
    """[n, 2] float32 numpy: the pixel centres of a 613 x 587 image stretched over the VAR_DET_LONG texture."""
    import numpy as np
    TH, TW = VAR_DET_LONG
    ys, xs = np.meshgrid(np.arange(613, dtype=np.float32), np.arange(587, dtype=np.float32), indexing='ij')
    rows = (ys + np.float32(0.5)) * np.float32(TH / 613.)
    cols = (xs + np.float32(0.5)) * np.float32(TW / 587.)
    return np.stack([rows.reshape(-1), cols.reshape(-1)], -1).astype(np.float32)


def normals_meshes():
    """name -> (vertices [V, 3], faces [F, 3]) numpy: an icosphere with 20 faces that name one vertex twice appended, and
    a fan of VAR_NORMALS_FAN faces around vertex 0 (a row longer than NORMALS_LONG_ROW, summed by a whole warp)."""
    import numpy as np
    from dirt_b200 import scenes
    v, f = scenes.icosphere(3)
    repeated = np.array([[f[i, 0], f[i, 0], f[i + 1, 1]] for i in range(0, 60, 3)], np.int32)
    n = VAR_NORMALS_FAN
    i = np.arange(n + 1)
    t = i * (np.pi * (3. - np.sqrt(5.)))
    rim = np.stack([np.cos(t), np.sin(t), -0.3 + 0.6 * i / n], axis=1)
    fan_v = np.concatenate([np.zeros((1, 3)), rim]).astype(np.float32)
    fan_f = np.stack([np.zeros(n), np.arange(1, n + 1), np.arange(2, n + 2)], axis=1).astype(np.int32)
    return {'icosphere': (v.astype(np.float32), np.concatenate([f, repeated]).astype(np.int32)), 'fan': (fan_v, fan_f)}


# (b) the product at its shipped limits
TEX_LOOKUPS = (1 << 24) + 4099
GENERIC_CHANNELS = [5, 6, 7]


def generic_lookups(C):
    """Lookups of the generic forward at C: their total * C just over 2^24 elements."""
    return (1 << 24) // C + 1001


MIP_SMALL = (256, 192)             # trilinear texture at TEX_LOOKUPS, read at levels 0 .. 3 (256x192 .. 32x24)
MIP_LARGE = (1, 4096, 2048, 9)     # a texture whose level 0 and level 1 take more than one round
MIP_LARGE_LOOKUPS = 1 << 16
DET_SCAN = ((61, 53), (1 << 20) + 3 * RS_TILE + 5)    # 260 sort tiles: two scan rounds
DET_PASSES = ((4097, 4096), 200003)                    # sentinel >= 2^24: four passes
DET_SLOTS = ((2, 2), 3 << 25)                          # 3 * 2^25 terms per texel: 98 304 chunk slots
LIGHT_B, LIGHT_V = 131077, 33
LIGHT_ITEMS = [0, 65534, 65535, 65536, 131070, LIGHT_B - 1]
# model: C.  Lambert's per-item parameters are 3 + C columns: C = 6 takes their total past 2^20 too
LIGHT_MODELS = {'diffuse_directional': 6, 'diffuse_point': 6, 'specular_directional': 3, 'ggx': 3, 'ggx_point': 3, 'sh': 3}
