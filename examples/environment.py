"""A mirror-and-diffuse sphere in front of a cube-map environment, through the deferred-shading entry point.

    python examples/environment.py [out.png]

The G-buffer holds [mask, normal, position] per pixel.  The background is `dirt_b200.sample_cubemap` of the view rays
that `projection.unproject_pixels_to_rays` gives for every pixel; the sphere shows the environment in the reflected view
vector, blended with a diffuse base colour.  The cube map is procedural (`procedural_cubemap`), so nothing is
downloaded.  Gradients reach the cube map (here, a toy loss), which is how an environment is fitted to photographs.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

frame_width, frame_height = 640, 480

# face -> the direction of face point (sc, tc): the inverse of the OpenGL cube-map table
_FACE_POINT = [lambda s, t: (1., -t, -s), lambda s, t: (-1., -t, s), lambda s, t: (s, 1., t),
               lambda s, t: (s, -1., -t), lambda s, t: (s, -t, 1.), lambda s, t: (-s, -t, -1.)]


def cubemap_directions(size, device=None):
    """Unit directions through the texel centres of a [6, size, size] cube map -> [6, size, size, 3]."""
    c = (torch.arange(size, dtype=torch.float32, device=device) + 0.5) / size * 2 - 1
    t, s = torch.meshgrid(c, c, indexing='ij')
    faces = []
    for point in _FACE_POINT:
        x, y, z = point(s, t)
        faces.append(torch.stack([torch.as_tensor(x, device=device).expand_as(s), torch.as_tensor(y, device=device).expand_as(s),
                                  torch.as_tensor(z, device=device).expand_as(s)], -1))
    d = torch.stack(faces)
    return d / d.norm(dim=-1, keepdim=True)


def sky(d):
    """An HDR-ish sky over a checkered ground, with a sun, in unit directions d [..., 3] -> [..., 3]."""
    device = d.device
    up = d[..., 1:2]
    sky = torch.tensor([0.25, 0.45, 0.9], device=device) * (0.6 + 0.4 * up) + 0.3 * (1 - up.abs())
    u, v = d[..., 0] / (d[..., 1].abs() + 0.2), d[..., 2] / (d[..., 1].abs() + 0.2)
    checks = (((u * 4).floor() + (v * 4).floor()) % 2)[..., None]
    ground = torch.tensor([0.35, 0.3, 0.25], device=device) * (0.5 + 0.5 * checks)
    sun_dir = torch.tensor([0.4, 0.6, -0.7], device=device)
    sun = 8.0 * torch.exp(-(1 - (d * (sun_dir / sun_dir.norm())).sum(-1, keepdim=True)) * 400.)
    return torch.where(up > 0, sky, ground) + sun


def procedural_cubemap(size=128, device=None):
    """`sky` at the texel centres of a cube map: [6, size, size, 3]."""
    return sky(cubemap_directions(size, device))


def sphere(level=4, device=None):
    """A unit icosphere: (vertices [V, 3], faces [F, 3] int32)."""
    from dirt_b200 import scenes
    v, f = scenes.icosphere(level)
    return torch.from_numpy(v).to(device), torch.from_numpy(f).to(device)


def camera(distance=3.2, width=frame_width, height=frame_height, device=None):
    """(view_projection [4, 4], camera position [3]): the camera at (0, 0, distance) looking at the origin."""
    from dirt_b200 import matrices
    view = matrices.translation([0., 0., -distance]).to(device)
    proj = matrices.perspective_projection(near=0.1, far=20., right=0.08, aspect=float(height) / width).to(device)
    return view @ proj, torch.tensor([0., 0., distance], device=device)


def background_rays(view_projection, width, height, batch=None):
    """The world-space view ray of every pixel centre [H, W, 3] ([B, H, W, 3] for a batch of matrices)."""
    from dirt_b200 import projection
    dev = view_projection.device
    ys, xs = torch.meshgrid(torch.arange(height, device=dev), torch.arange(width, device=dev), indexing='ij')
    pixels = torch.stack([xs, ys], -1).to(torch.float32) + 0.5
    size = torch.tensor([float(width), float(height)], device=dev)
    if batch is not None:
        pixels, size = pixels.expand(batch, height, width, 2), size.expand(batch, 2)
    _, rays = projection.unproject_pixels_to_rays(pixels, torch.linalg.inv(view_projection), size)
    return rays


def shader_fn(gbuffer, cubemap, rays, camera_position, base_colour, sample, mirror=0.7):
    """G-buffer [..., H, W, 7] = (mask, normal, position) -> pixels [..., H, W, 3]: a mirror reflection of the cube map
    blended with a diffuse base colour lit by the cube map's value along the normal, over the cube map behind.
    `sample`: `dirt_b200.sample_cubemap`, or any lookup with its signature."""
    mask, normals, positions = gbuffer[..., :1], gbuffer[..., 1:4], gbuffer[..., 4:7]
    view = positions - camera_position
    view = view / view.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    reflected = view - 2. * (view * normals).sum(-1, keepdim=True) * normals
    # the lookups of pixels off the sphere: any direction; their values are masked out below
    reflection = sample(cubemap, torch.where(mask > 0, reflected, rays))
    diffuse = sample(cubemap, torch.where(mask > 0, normals, rays))
    surface = mirror * reflection + (1. - mirror) * base_colour * diffuse
    return surface * mask + sample(cubemap, rays) * (1. - mask)


def render(cubemap, rasterise, sample, batch=None, width=frame_width, height=frame_height, device=None):
    """The sphere in front of `cubemap` ([6, S, S, 3], or [B, 6, S, S, 3] with `batch`) -> pixels."""
    vertices, faces = sphere(device=device)
    view_projection, eye = camera(width=width, height=height, device=device)
    clip = torch.cat([vertices, torch.ones_like(vertices[:, :1])], 1) @ view_projection
    attributes = torch.cat([torch.ones_like(vertices[:, :1]), vertices, vertices], 1)   # unit sphere: normal = position
    base = torch.tensor([0.8, 0.3, 0.2], device=device)
    if batch is None:
        rays = background_rays(view_projection, width, height)
        return rasterise(torch.zeros(height, width, 7, device=device), clip, attributes, faces,
                         lambda gb, cm: shader_fn(gb, cm, rays, eye, base, sample), [cubemap])
    rays = background_rays(view_projection.expand(batch, 4, 4), width, height, batch)
    return rasterise(torch.zeros(batch, height, width, 7, device=device), clip.expand(batch, -1, -1),
                     attributes.expand(batch, -1, -1), faces.expand(batch, -1, -1),
                     lambda gb, cm: shader_fn(gb, cm, rays, eye, base, sample), [cubemap])


def main():
    import dirt_b200 as dirt
    device = torch.device('cuda')
    cubemap = procedural_cubemap(device=device).requires_grad_(True)
    pixels = render(cubemap, dirt.rasterise_deferred, dirt.sample_cubemap, device=device)
    loss = pixels.mean()   # a toy loss: the gradient reaches the texels behind the background and in the reflection
    loss.backward()
    print('rendered %dx%d; d loss / d cube map touches %d of %d texels'
          % (frame_width, frame_height, int((cubemap.grad.abs().sum(-1) > 0).sum()), cubemap.shape[0] * cubemap.shape[1] ** 2))
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
