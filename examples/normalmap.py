"""A normal-mapped sphere under several lights, and a photometric-stereo fit of its normal map through the renderer.

    python examples/normalmap.py

The sphere has a seam column: its seam vertices are split, so each side of the seam has its own uvs.  Its tangent
frames come from `lighting.vertex_tangents`, and it is rendered through `rasterise_batch_deferred` into a G-buffer of
[mask, uv, normal, tangent, position] (13 channels).  The shader reads a tangent-space normal map with `sample_texture`
(trilinear, its level of detail from the exact uv derivatives of `derivative_channels`), perturbs the normals with
`lighting.perturb_normals` and lights them with `diffuse_directional` plus `specular_ggx_directional`, one light
direction per batch item.  `main` fits the normal map, from a flat start, to renders of a procedural one made from a
height field, and prints the image loss before and after.
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))


def seamed_sphere(columns=64, rows=32, device=None):
    """A unit uv sphere with columns + 1 vertices per ring: the last of each ring is a copy of the first, with u = 1.
    Returns positions [V, 3], uvs [V, 2] (u along the longitude, v from the north pole down) and int32 faces [F, 3]."""
    u = torch.arange(columns + 1, dtype=torch.float64) / columns
    v = torch.arange(rows + 1, dtype=torch.float64) / rows
    vv, uu = torch.meshgrid(v, u, indexing='ij')
    phi, theta = 2 * math.pi * uu, math.pi * vv
    p = torch.stack([theta.sin() * phi.sin(), theta.cos(), theta.sin() * phi.cos()], -1).reshape(-1, 3)
    uv = torch.stack([uu, vv], -1).reshape(-1, 2)
    i = torch.arange(rows)[:, None] * (columns + 1) + torch.arange(columns)[None, :]
    a, b, c, d = i, i + 1, i + columns + 1, i + columns + 2
    # the first row's (a, c, b) and the last row's (b, c, d) would have two corners at a pole
    faces = torch.cat([torch.stack([a, c, b], -1)[1:].reshape(-1, 3), torch.stack([b, c, d], -1)[:-1].reshape(-1, 3)])
    return (p.to(torch.float32).to(device), uv.to(torch.float32).to(device),
            faces.to(torch.int32).to(device))


def height_normal_map(size=64, strength=0.6, device=None):
    """A tangent-space normal map [size, size, 3] encoded to [0, 1], made from the height field
    h = sum of sinusoidal bumps in (u, v): n = unit(-k dh/du, -k dh/dv, 1).  Row r, column c is (v, u) = (r, c) / size,
    the convention of `texture.uvs_to_pixel_indices`."""
    r = (torch.arange(size, device=device, dtype=torch.float32) + 0.5) / size
    v, u = torch.meshgrid(r, r, indexing='ij')
    two_pi = 2 * math.pi
    dh_du = two_pi * 4 * torch.cos(two_pi * 4 * u) * torch.sin(two_pi * 3 * v) + two_pi * 2 * torch.cos(two_pi * 2 * (u + v))
    dh_dv = two_pi * 3 * torch.sin(two_pi * 4 * u) * torch.cos(two_pi * 3 * v) + two_pi * 2 * torch.cos(two_pi * 2 * (u + v))
    k = strength / (two_pi * 4)
    n = torch.nn.functional.normalize(torch.stack([-k * dh_du, -k * dh_dv, torch.ones_like(u)], -1), dim=-1)
    return 0.5 * (n + 1.)


def shader_fn(gbuffer, normal_map, light_directions, camera_position, gbuffer_derivatives):
    """G-buffer [B, H, W, 13] = (mask, uv, normal, tangent, position) -> pixels [B, H, W, 3]; normal_map [S, S, 3]
    encoded to [0, 1]; light_directions [B, 3]; gbuffer_derivatives [B, H, W, 2, 2] of the uv channels."""
    from dirt_b200 import lighting
    from dirt_b200.texture import sample_texture, uvs_to_pixel_indices
    B, H, W, _ = gbuffer.shape
    S = normal_map.shape[0]
    mask, uv = gbuffer[..., :1], gbuffer[..., 1:3]
    rows = lambda a, b: gbuffer[..., a:b].reshape(B, H * W, b - a)   # views of the G-buffer, read in place
    # uv per pixel -> (row, column) texel indices per pixel: row = v S, column = u S
    d = gbuffer_derivatives * S
    derivatives = torch.stack([d[..., 0, 1], d[..., 0, 0], d[..., 1, 1], d[..., 1, 0]], -1)
    m = 2. * sample_texture(normal_map, uvs_to_pixel_indices(uv, (S, S)), 'trilinear', derivatives) - 1.
    n = lighting.perturb_normals(rows(3, 6), rows(6, 10), m.reshape(B, H * W, 3))
    p = rows(10, 13)
    albedo = torch.tensor([0.7, 0.6, 0.5], device=gbuffer.device).expand(B, H * W, 3)
    light_color = torch.ones(3, device=gbuffer.device)
    diffuse = lighting.diffuse_directional(n, albedo, light_directions, light_color, double_sided=False)
    specular = lighting.specular_ggx_directional(p, n, torch.full((B, H * W, 1), 0.35, device=gbuffer.device),
                                                 torch.full((B, H * W, 3), 0.04, device=gbuffer.device),
                                                 light_directions, light_color, camera_position)
    return (diffuse + specular).reshape(B, H, W, 3) * mask


def render(normal_map, light_directions, size=128):
    """The sphere, normal-mapped with `normal_map`, under each of light_directions [B, 3]: [B, size, size, 3]."""
    import dirt_b200 as dirt
    from dirt_b200 import lighting, matrices
    device = normal_map.device
    B = light_directions.shape[0]
    p, uv, faces = seamed_sphere(device=device)
    n = lighting.vertex_normals(p, faces)
    t = lighting.vertex_tangents(p, uv, faces, n)
    eye = torch.tensor([0., 0., 3.], device=device)
    view = matrices.translation([0., 0., -3.]).to(device)
    proj = matrices.perspective_projection(near=0.1, far=20., right=0.05, aspect=1.).to(device)
    clip = torch.cat([p, torch.ones_like(p[:, :1])], 1) @ view @ proj
    attributes = torch.cat([torch.ones_like(p[:, :1]), uv, n, t, p], 1)   # 13 channels
    return dirt.rasterise_batch_deferred(
        torch.zeros(B, size, size, 13, device=device), clip.expand(B, -1, -1), attributes.expand(B, -1, -1),
        faces.expand(B, -1, -1),
        lambda gb, nm, gbuffer_derivatives: shader_fn(gb, nm, light_directions, eye, gbuffer_derivatives), [normal_map],
        derivative_channels=range(1, 3))


def fit_normal_map(target_map, light_directions, steps=150, lr=0.05, size=128):
    """Fits a normal map from a flat start to the renders of `target_map` with Adam.  Returns (map, losses)."""
    with torch.no_grad():
        target = render(target_map, light_directions, size)
    flat = torch.tensor([0.5, 0.5, 1.], device=target_map.device)
    normal_map = flat.expand(target_map.shape).clone().requires_grad_(True)
    opt = torch.optim.Adam([normal_map], lr=lr)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = ((render(normal_map, light_directions, size) - target) ** 2).mean()
        loss.backward()
        opt.step()
        with torch.no_grad():
            normal_map.clamp_(0., 1.)
        losses.append(float(loss.detach()))
    with torch.no_grad():
        losses.append(float(((render(normal_map, light_directions, size) - target) ** 2).mean()))
    return normal_map.detach(), losses


def main(steps=150, size=128, verbose=True):
    """Returns the image loss before and after the fit."""
    device = torch.device('cuda')
    lights = torch.nn.functional.normalize(torch.tensor([[0.6, -0.4, -1.], [-0.7, -0.3, -1.], [0.1, 0.8, -1.],
                                                         [0.2, -0.9, -0.6]], device=device), dim=-1)
    truth = height_normal_map(device=device)
    _, losses = fit_normal_map(truth, lights, steps=steps, size=size)
    if verbose:
        print('normal-map fit, %d lights, %d steps: image loss %.5f -> %.5f' % (lights.shape[0], steps, losses[0],
                                                                               losses[-1]))
    return losses[0], losses[-1]


if __name__ == '__main__':
    main()
