"""Spheres lit by one cube-map environment through split-sum GGX image-based lighting, and fits through the renderer.

    python examples/ibl.py

Each sphere is rendered through `rasterise_batch_deferred`: GGX specular from `lighting.specular_ggx_environment`
(the cube map prefiltered with the GGX lobe, `sample_cubemap(..., mode='ggx')`, times the split-sum BRDF) plus
Lambertian diffuse from `lighting.diffuse_spherical_harmonics` of `lighting.cubemap_spherical_harmonics` of the same
map, over the map itself behind.  `fit_material` recovers per-item roughness and specular colour (F0) from rendered
images with Adam; `fit_environment` fits a 16 x 16 environment from the images of known materials.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

import environment as env   # noqa: E402


def shader_fn(gbuffer, cubemap, roughness, f0, rays, camera_position, albedo):
    """G-buffer [B, H, W, 7] = (mask, normal, position) -> pixels [B, H, W, 3]; cubemap [B, 6, S, S, 3], roughness
    [B], f0 [B, 3]."""
    from dirt_b200 import lighting
    import dirt_b200 as dirt
    B, H, W, _ = gbuffer.shape
    mask, normals, positions = gbuffer[..., :1], gbuffer[..., 1:4], gbuffer[..., 4:7]
    n, p = normals.reshape(B, H * W, 3), positions.reshape(B, H * W, 3)
    rough = roughness[:, None, None].expand(B, H * W, 1)
    spec = lighting.specular_ggx_environment(p, n, rough, f0[:, None, :].expand(B, H * W, 3), cubemap, camera_position)
    diffuse = lighting.diffuse_spherical_harmonics(n, albedo.expand(B, H * W, 3), lighting.cubemap_spherical_harmonics(cubemap))
    surface = (spec + diffuse).reshape(B, H, W, 3)
    return surface * mask + dirt.sample_cubemap(cubemap, rays, 'bilinear') * (1. - mask)


def render(cubemap, roughness, f0, batch, width=128, height=96):
    """Spheres in front of `cubemap` [B, 6, S, S, 3], one per item, with roughness [B] and F0 [B, 3]."""
    import dirt_b200 as dirt
    device = cubemap.device
    vertices, faces = env.sphere(device=device)
    view_projection, eye = env.camera(width=width, height=height, device=device)
    clip = torch.cat([vertices, torch.ones_like(vertices[:, :1])], 1) @ view_projection
    attributes = torch.cat([torch.ones_like(vertices[:, :1]), vertices, vertices], 1)   # unit sphere: normal = position
    albedo = torch.tensor([0.6, 0.35, 0.25], device=device)
    rays = env.background_rays(view_projection.expand(batch, 4, 4), width, height, batch)
    return dirt.rasterise_batch_deferred(
        torch.zeros(batch, height, width, 7, device=device), clip.expand(batch, -1, -1), attributes.expand(batch, -1, -1),
        faces.expand(batch, -1, -1), lambda gb, cm, ro, f: shader_fn(gb, cm, ro, f, rays, eye, albedo),
        [cubemap, roughness, f0])


def fit_material(cubemap, truth_roughness, truth_f0, start_roughness, start_f0, steps=300, lr=0.03):
    """Per-item roughness [B] and F0 [B, 3] fitted with Adam from the start values to images rendered at the truth.
    Returns (roughness, f0) after each step, [steps + 1, B] and [steps + 1, B, 3]."""
    B = truth_roughness.shape[0]
    with torch.no_grad():
        target = render(cubemap, truth_roughness, truth_f0, B)
    roughness = start_roughness.detach().clone().requires_grad_(True)
    f0 = start_f0.detach().clone().requires_grad_(True)
    opt = torch.optim.Adam([roughness, f0], lr=lr)
    path_r, path_f = [roughness.detach().clone()], [f0.detach().clone()]
    for _ in range(steps):
        opt.zero_grad()
        ((render(cubemap, roughness, f0, B) - target) ** 2).mean().backward()
        opt.step()
        with torch.no_grad():
            roughness.clamp_(0.05, 1.)
            f0.clamp_(0., 1.)
        path_r.append(roughness.detach().clone())
        path_f.append(f0.detach().clone())
    return torch.stack(path_r), torch.stack(path_f)


def fit_environment(truth_cubemap, roughness, f0, steps=100, lr=0.05, size=16):
    """A size x size environment, shared by the items, fitted with Adam from a uniform grey to images rendered in
    `truth_cubemap` [6, S, S, 3] with known materials.  Returns (loss before, loss after)."""
    B = roughness.shape[0]
    with torch.no_grad():
        target = render(truth_cubemap.expand(B, -1, -1, -1, -1).contiguous(), roughness, f0, B)
    cube = torch.full((6, size, size, 3), 0.5, device=truth_cubemap.device, requires_grad=True)
    opt = torch.optim.Adam([cube], lr=lr)
    losses = []
    for _ in range(steps + 1):
        opt.zero_grad()
        loss = ((render(cube.expand(B, -1, -1, -1, -1), roughness, f0, B) - target) ** 2).mean()
        losses.append(float(loss))
        loss.backward()
        opt.step()
    return losses[0], losses[-1]


def main():
    device = torch.device('cuda')
    cubemap = env.procedural_cubemap(64, device=device)
    B = 2
    cubes = cubemap.expand(B, -1, -1, -1, -1).contiguous()
    truth_r, truth_f = torch.tensor([0.3, 0.55], device=device), torch.tensor([[0.9, 0.6, 0.3], [0.3, 0.3, 0.3]],
                                                                             device=device)
    start_r, start_f = torch.tensor([0.8, 0.1], device=device), torch.full((B, 3), 0.5, device=device)
    path_r, path_f = fit_material(cubes, truth_r, truth_f, start_r, start_f)
    print('fitted roughness %s -> %s (truth %s)' % (start_r.tolist(), [round(x, 4) for x in path_r[-1].tolist()],
                                                    truth_r.tolist()))
    print('fitted F0 %s -> %s (truth %s)' % (start_f.tolist(), [[round(x, 4) for x in r] for r in path_f[-1].tolist()],
                                             truth_f.tolist()))
    before, after = fit_environment(cubemap, truth_r, truth_f)
    print('16 x 16 environment fit: image loss %.4g -> %.4g' % (before, after))


if __name__ == '__main__':
    main()
