"""The split-sum GGX environment lookup of sample_cubemap(..., mode='ggx', roughness=...) and its BRDF table
(DESIGN.md §7.12) restated in numpy and torch.  It is the specification of the prefiltered levels and of the table; the
CUDA lookup on given levels equals cubemap_mip_restatement's level blend of them bit for bit.

    levels      L = level_count(S); level 0 is the cube map; level k >= 1, S_k = S >> k per edge, is the GGX prefilter
                of box level s_k = min(k, s*) (cubemap_mip_restatement.pyramid), s* the coarsest level with at least 16
                texels per edge (0 when S < 16), at roughness r_k = k / (L-1)
    lobe        a = max(r_k, 0.045), alpha2 = a^4 (float64, then rounded once to fp32 for the kernel);
                c_k = max(0, 1 - 2 (sqrt(1000) - 1) alpha2 / (1 - alpha2)) in float64 (0 where alpha2 = 1), rounded
                once to fp32: the texels whose D is at least 1e-3 of the lobe's peak
    texels      per level, face f, row r, column c: sc = (2c+1)/S_k - 1, tc = (2r+1)/S_k - 1 in fp32; (x, y, z) by the
                face table of cubemap_restatement.border_source; n = sqrt(fma(z, z, fma(y, y, x*x))); direction
                (x/n, y/n, z/n), each operation rounded in fp32 in that order.  Solid angle: the corner formula
                sum +- atan2(u v, sqrt(u^2 + v^2 + 1)) over the texel's corners (u, v) in float64, rounded once to fp32
    pairs       c = fma(r.z, l.z, fma(r.y, l.y, r.x * l.x)) in fp32 (symmetric in r and l); source texel l is in the
                sum of output texel r iff c > 0 and c >= c_k (the same fp32 decision as the kernel's)
    sum         P_k(r) = sum_j w_j src_j / W(r), W(r) = sum_j w_j, w_j = D(c_j) c_j Omega_j, D(c) = alpha2 / (pi k^2),
                k = alpha2 + (1 - c)(1 - alpha2)/2; here in float64 (the kernel's fp32 sums are compared within a
                tolerance)
    lookup      lod = roughness * (L-1), then cubemap_mip_restatement.blend of the bilinear reads of the levels
    BRDF table  (A, B) at n.v = (i + 0.5)/N, roughness (j + 0.5)/N: the midpoint rule of `brdf_node`, over
                u = 1 - t^2 of the GGX half-vector distribution's inverse (weight 2t) and phi."""
import math

import numpy as np
import torch

import cubemap_mip_restatement as cmm
import cubemap_restatement as cm

MIN_ROUGHNESS = 0.045
BRDF_N, BRDF_U, BRDF_PHI = 128, 1024, 64


def level_count(S):
    return cmm.level_count(S)


def source_cap(S):
    """s*: the coarsest level with at least 16 texels per edge, 0 when S < 16."""
    ss = 0
    for k in range(level_count(S)):
        if (S >> k) >= 16:
            ss = k
    return ss


def lobe(k, L):
    """(alpha2 float64, alpha2 fp32, c_k fp32) of level k >= 1."""
    r = k / (L - 1)
    a = max(r, MIN_ROUGHNESS)
    alpha2 = (a * a) * (a * a)
    ck = 0.0 if alpha2 >= 1.0 else 1.0 - 2.0 * (math.sqrt(1000.0) - 1.0) * alpha2 / (1.0 - alpha2)
    return alpha2, np.float32(alpha2), np.float32(max(ck, 0.0))


def fmaf(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: the exact product in float64, an error-free sum, and one rounding to fp32
    that settles float64's ties by the sum's remainder."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b                                  # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)              # s + e == p + c exactly
    f = s.astype(np.float32)
    lo = np.where(f.astype(np.float64) > s, np.nextafter(f, np.float32(-np.inf)), f)
    hi = np.nextafter(lo, np.float32(np.inf))
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) * 0.5
    tie = (s == mid) & (e != 0)
    return np.where(tie, np.where(e > 0, hi, lo), f).astype(np.float32)


def _face_point(f, sc, tc):
    one = np.ones_like(sc)
    return [(one, -tc, -sc), (-one, -tc, sc), (sc, one, tc), (sc, -one, -tc), (sc, -tc, one), (-sc, -tc, -one)][f]


_TABLES = {}


def texel_table(S):
    """(directions fp32 [6, S, S, 3], solid angles fp32 [6, S, S]) of a level of S texels per edge."""
    if S not in _TABLES:
        i = np.arange(S)
        Sf = np.float32(S)
        centre = (np.float32(2) * i.astype(np.float32) + np.float32(1)) / Sf - np.float32(1)
        tc, sc = np.meshgrid(centre.astype(np.float32), centre.astype(np.float32), indexing='ij')
        dirs = np.zeros((6, S, S, 3), np.float32)
        edge = 2.0 * np.arange(S + 1) / S - 1.0
        F = lambda u, v: np.arctan2(u * v, np.sqrt(u * u + v * v + 1.0))
        v0, u0 = np.meshgrid(edge[:-1], edge[:-1], indexing='ij')
        v1, u1 = np.meshgrid(edge[1:], edge[1:], indexing='ij')
        omega = (F(u1, v1) - F(u0, v1) - F(u1, v0) + F(u0, v0)).astype(np.float32)
        for f in range(6):
            x, y, z = (np.asarray(t, np.float32) for t in _face_point(f, sc, tc))
            n = np.sqrt(fmaf(z, z, fmaf(y, y, x * x)))
            dirs[f] = np.stack([x / n, y / n, z / n], -1)
        _TABLES[S] = (dirs, np.broadcast_to(omega, (6, S, S)).copy())
    return _TABLES[S]


def pair_cos(r, l):
    """fp32 c = fma(r.z, l.z, fma(r.y, l.y, r.x * l.x)) of every pair: r [n, 3], l [m, 3] -> [n, m]."""
    r, l = r[:, None, :], l[None, :, :]
    return fmaf(r[..., 2], l[..., 2], fmaf(r[..., 1], l[..., 1], r[..., 0] * l[..., 0]))


def support(r, l, ck):
    c = pair_cos(r, l)
    return c, (c > 0) & (c >= ck)


_WEIGHTS = {}


def weights(k, L, S, chunk=1024):
    """Level k's pair weights, float64 [6 S_k^2, 6 S_s^2] (0 outside the support), and s_k (kept per (k, L, S))."""
    if (k, L, S) not in _WEIGHTS:
        _WEIGHTS[(k, L, S)] = _weights(k, L, S, chunk)
    return _WEIGHTS[(k, L, S)]


def _weights(k, L, S, chunk):
    s = min(k, source_cap(S))
    alpha2, _, ck = lobe(k, L)
    rd, _ = texel_table(S >> k)
    ld, lw = texel_table(S >> s)
    rd, ld, lw = rd.reshape(-1, 3), ld.reshape(-1, 3), lw.reshape(-1).astype(np.float64)
    out = np.zeros((rd.shape[0], ld.shape[0]))
    for a in range(0, rd.shape[0], chunk):
        c, keep = support(rd[a:a + chunk], ld, ck)
        c = c.astype(np.float64)
        kk = alpha2 + (1.0 - c) * (1.0 - alpha2) / 2.0
        out[a:a + chunk] = np.where(keep, alpha2 / (math.pi * kk * kk) * c * lw, 0.0)
    return out, s


def prefiltered_levels(cubemap):
    """[6, S, S, C] -> levels 0 .. L-1, each [6, S_k, S_k, C], in cubemap's dtype (float64 for the specification);
    differentiable in cubemap."""
    S = cubemap.shape[-2]
    L = level_count(S)
    box = cmm.pyramid(cubemap)
    levels = [cubemap]
    for k in range(1, L):
        w, s = weights(k, L, S)
        w = torch.as_tensor(w, dtype=cubemap.dtype, device=cubemap.device)
        src = box[s].reshape(-1, cubemap.shape[-1])
        P = (w @ src) / w.sum(1, keepdim=True)
        levels.append(P.reshape(6, S >> k, S >> k, cubemap.shape[-1]))
    return levels


def normalisers(S):
    """W of levels 1 .. L-1, float64 [6, S_k, S_k] each."""
    L = level_count(S)
    return [weights(k, L, S)[0].sum(1).reshape(6, S >> k, S >> k) for k in range(1, L)]


def blend_levels(levels, directions, lod, coords_of=None):
    """cubemap_mip_restatement's lookup on the given levels: [..., 3] directions, lod [...] -> [..., C]."""
    reads = []
    for k, level in enumerate(levels):
        face, s, t, valid = (coords_of or (lambda d, k, S: cm.face_coords(d)))(directions, k, level.shape[-2])
        reads.append(cm.sample_padded(cm.atlas(level), face, s, t, valid, 'bilinear'))
    return cmm.blend(reads, lod, cm.face_coords(directions)[3])


def sample(cubemap, directions, roughness, coords_of=None):
    """cubemap [6, S, S, C] with directions [..., 3] and roughness [...], or [B, 6, S, S, C] with [B, ..., 3] and
    [B, ...] -> [..., C]."""
    if cubemap.dim() == 5:
        return torch.stack([sample(cubemap[b], directions[b], roughness[b], coords_of) for b in range(cubemap.shape[0])])
    lod = roughness * float(level_count(cubemap.shape[-2]) - 1)
    return blend_levels(prefiltered_levels(cubemap), directions, lod, coords_of)


def brdf_node(n_dot_v, roughness, U=BRDF_U, PHI=BRDF_PHI):
    """(A, B), float64, by the table kernel's midpoint rule over the GGX half-vector distribution."""
    a = max(roughness, MIN_ROUGHNESS)
    alpha2 = (a * a) * (a * a)
    nv = n_dot_v
    vx, vz = math.sqrt(1.0 - nv * nv), nv
    t = (np.arange(U) + 0.5) / U
    x = 1.0 - t * t   # u = 1 - t^2: the integrand's 1 / sqrt(1 - u) at grazing half-vectors becomes smooth in t
    ch = np.sqrt((1.0 - x) / (1.0 + (alpha2 - 1.0) * x))
    sh = np.sqrt(np.maximum(0.0, 1.0 - ch * ch))
    phi = 2.0 * math.pi * (np.arange(PHI) + 0.5) / PHI
    ch, sh, phi, t = ch[:, None], sh[:, None], phi[None, :], t[:, None]
    hx, hz = sh * np.cos(phi), ch
    vh = vx * hx + vz * hz
    nl = 2.0 * vh * hz - vz
    ok = (nl > 0) & (vh > 0)
    nl_ = np.where(ok, nl, 1.0)
    vis = 0.5 / (nl_ * math.sqrt(nv * nv * (1.0 - alpha2) + alpha2) + nv * np.sqrt(nl_ * nl_ * (1.0 - alpha2) + alpha2))
    g = np.where(ok, vis * nl_ * 4.0 * vh / ch * (2.0 * t), 0.0)
    m = 1.0 - vh
    fc = (m * m) * (m * m) * m
    return float(((1.0 - fc) * g).sum() / (U * PHI)), float((fc * g).sum() / (U * PHI))


def sh_project(cubemap):
    """[6, S, S, C] -> [9, C]: sum_j L(l_j) Y_k(l_j) Omega_j over level 0's texel table, lighting._sh_basis, in cubemap's
    dtype; differentiable in cubemap."""
    from dirt_b200 import lighting
    dirs, omega = texel_table(cubemap.shape[-2])
    d = torch.as_tensor(dirs.reshape(-1, 3), dtype=cubemap.dtype, device=cubemap.device)
    w = torch.as_tensor(omega.reshape(-1), dtype=cubemap.dtype, device=cubemap.device)
    Y = lighting._sh_basis(d)                                     # [n, 9]
    return (Y * w[:, None]).T @ cubemap.reshape(-1, cubemap.shape[-1])
