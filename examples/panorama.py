"""An equirectangular (latitude-longitude) environment: converted to a cube map for image-based lighting, and fitted.

    python examples/panorama.py

Builds a procedural panorama, `environment.sky` evaluated at `latlong_directions`, renders the spheres of
examples/ibl.py lit by `latlong_to_cubemap` of it, and fits a 32 x 64 panorama from a uniform grey to those images
through the renderer with the materials known.  The fitted panorama is the parameter: the conversion runs on every
step, and its gradient reaches the panorama's texels.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

import environment as env   # noqa: E402
import ibl                  # noqa: E402


def procedural_panorama(height=256, width=512, device=None):
    """`environment.sky` at the texel centres of a [height, width] panorama -> [height, width, 3]."""
    import dirt_b200 as dirt
    return env.sky(dirt.latlong_directions(height, width, device=device))


def fit_panorama(truth_panorama, roughness, f0, height=32, width=64, size=16, steps=100, lr=0.05):
    """A height x width panorama, shared by the items, fitted with Adam from a uniform grey to images of spheres lit
    by `truth_panorama` with known materials; the renderer reads it through a size x size cube map.  Returns
    (loss before, loss after)."""
    import dirt_b200 as dirt
    B = roughness.shape[0]
    with torch.no_grad():
        truth = dirt.latlong_to_cubemap(truth_panorama, 64)
        target = ibl.render(truth.expand(B, -1, -1, -1, -1).contiguous(), roughness, f0, B)
    panorama = torch.full((height, width, 3), 0.5, device=truth_panorama.device, requires_grad=True)
    opt = torch.optim.Adam([panorama], lr=lr)
    losses = []
    for _ in range(steps + 1):
        opt.zero_grad()
        cube = dirt.latlong_to_cubemap(panorama, size)
        loss = ((ibl.render(cube.expand(B, -1, -1, -1, -1), roughness, f0, B) - target) ** 2).mean()
        losses.append(float(loss.detach()))
        loss.backward()
        opt.step()
    return losses[0], losses[-1]


def main():
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    device = torch.device('cuda')
    panorama = procedural_panorama(device=device)
    H, W = panorama.shape[:2]
    cube = dirt.latlong_to_cubemap(panorama, 64)
    B = 2
    roughness = torch.tensor([0.3, 0.55], device=device)
    f0 = torch.tensor([[0.9, 0.6, 0.3], [0.3, 0.3, 0.3]], device=device)
    pixels = ibl.render(cube.expand(B, -1, -1, -1, -1).contiguous(), roughness, f0, B)
    n = _lib.lib().dirt_latlong_samples(H, W, 64)
    print('panorama %d x %d -> cube map 6 x 64 x 64, %d x %d samples per texel; %d spheres rendered, mean %.4f'
          % (H, W, n, n, B, float(pixels.mean())))
    before, after = fit_panorama(panorama, roughness, f0)
    print('32 x 64 panorama fit: image loss %.4g -> %.4g' % (before, after))


if __name__ == '__main__':
    main()
