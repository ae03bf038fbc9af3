"""A glossy sphere in front of a cube-map environment: the reflection blurred by a roughness, through the mip pyramid.

    python examples/glossy.py [out.png]

As examples/environment.py (whose scene helpers it uses), but the reflection reads
`dirt_b200.sample_cubemap(..., mode='trilinear', lod=...)` at a level of detail mapped from a roughness
(`roughness_to_lod`), and the diffuse term reads the coarsest level, the mean of each face, as a cheap irradiance.
`lod` is differentiable, so the roughness itself can be fitted through the renderer: `fit_roughness` recovers it from
rendered images.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

import environment as env   # noqa: E402

frame_width, frame_height = 640, 480


def levels(size):
    """The levels of a cube map of `size` texels per edge (dirt_texture_mip_levels's rule)."""
    L = 1
    while size % 2 == 0:
        size, L = size // 2, L + 1
    return L


def roughness_to_lod(roughness, size):
    """Roughness in [0, 1] -> level of detail: 0 (the sharp map) at roughness 0, the coarsest level at 1.  The blur of
    level k is 2^k texels, so the lod grows with log2 of the lobe width; a linear map is close enough for a demo."""
    return roughness * float(levels(size) - 1)


def shader_fn(gbuffer, cubemap, lod, rays, camera_position, base_colour, sample, specular=0.7):
    """G-buffer [..., H, W, 7] = (mask, normal, position) -> pixels [..., H, W, 3]: the cube map's reflection at level of
    detail `lod` (a float, or a tensor broadcastable to [..., H, W]) blended with a diffuse base colour lit by the
    coarsest level along the normal, over the sharp cube map behind."""
    mask, normals, positions = gbuffer[..., :1], gbuffer[..., 1:4], gbuffer[..., 4:7]
    view = positions - camera_position
    view = view / view.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    reflected = view - 2. * (view * normals).sum(-1, keepdim=True) * normals
    coarsest = float(levels(cubemap.shape[-2]) - 1)
    reflection = sample(cubemap, torch.where(mask > 0, reflected, rays), 'trilinear', lod=lod)
    irradiance = sample(cubemap, torch.where(mask > 0, normals, rays), 'trilinear', lod=coarsest)
    surface = specular * reflection + (1. - specular) * base_colour * irradiance
    return surface * mask + sample(cubemap, rays, 'bilinear') * (1. - mask)


def render(cubemap, roughness, rasterise, sample, batch=None, width=frame_width, height=frame_height, device=None):
    """The glossy sphere in front of `cubemap` ([6, S, S, 3], or [B, 6, S, S, 3] with `batch`, then `roughness` [B])."""
    vertices, faces = env.sphere(device=device)
    view_projection, eye = env.camera(width=width, height=height, device=device)
    clip = torch.cat([vertices, torch.ones_like(vertices[:, :1])], 1) @ view_projection
    attributes = torch.cat([torch.ones_like(vertices[:, :1]), vertices, vertices], 1)   # unit sphere: normal = position
    base = torch.tensor([0.8, 0.3, 0.2], device=device)
    lod = roughness_to_lod(torch.as_tensor(roughness, dtype=torch.float32, device=device), cubemap.shape[-2])
    if batch is None:
        rays = env.background_rays(view_projection, width, height)
        return rasterise(torch.zeros(height, width, 7, device=device), clip, attributes, faces,
                         lambda gb, cm, lo: shader_fn(gb, cm, lo, rays, eye, base, sample), [cubemap, lod])
    rays = env.background_rays(view_projection.expand(batch, 4, 4), width, height, batch)
    return rasterise(torch.zeros(batch, height, width, 7, device=device), clip.expand(batch, -1, -1),
                     attributes.expand(batch, -1, -1), faces.expand(batch, -1, -1),
                     lambda gb, cm, lo: shader_fn(gb, cm, lo[:, None, None], rays, eye, base, sample), [cubemap, lod])


def fit_roughness(cubemap, truth, start, rasterise, sample, steps=150, lr=0.03, width=128, height=96):
    """Per-item roughness fitted with Adam from `start` to images rendered at `truth` (both [B]).  Returns the
    roughness after each step, [steps + 1, B]."""
    B = truth.shape[0]
    with torch.no_grad():
        target = render(cubemap, truth, rasterise, sample, batch=B, width=width, height=height, device=cubemap.device)
    roughness = start.detach().clone().requires_grad_(True)
    opt = torch.optim.Adam([roughness], lr=lr)
    path = [roughness.detach().clone()]
    for _ in range(steps):
        opt.zero_grad()
        pixels = render(cubemap, roughness, rasterise, sample, batch=B, width=width, height=height, device=cubemap.device)
        ((pixels - target) ** 2).mean().backward()
        opt.step()
        with torch.no_grad():
            roughness.clamp_(0., 1.)
        path.append(roughness.detach().clone())
    return torch.stack(path)


def main():
    import dirt_b200 as dirt
    device = torch.device('cuda')
    cubemap = env.procedural_cubemap(128, device=device)
    pixels = render(cubemap, 0.4, dirt.rasterise_deferred, dirt.sample_cubemap, device=device)
    B = 2
    cubes = cubemap.expand(B, -1, -1, -1, -1).contiguous()
    truth, start = torch.tensor([0.35, 0.6], device=device), torch.tensor([0.8, 0.15], device=device)
    path = fit_roughness(cubes, truth, start, dirt.rasterise_batch_deferred, dirt.sample_cubemap)
    print('rendered %dx%d; fitted roughness %s -> %s (truth %s)'
          % (frame_width, frame_height, start.tolist(), [round(x, 4) for x in path[-1].tolist()], truth.tolist()))
    out = sys.argv[1] if len(sys.argv) > 1 else None
    if out:
        try:
            import cv2
            cv2.imwrite(out, (pixels.detach().clamp(0, 1) * 255).byte().cpu().numpy()[:, :, ::-1])
            print('wrote', out)
        except ImportError:
            print('cv2 not available; image not written')


if __name__ == '__main__':
    main()
