"""Seeded meshes of the timing scripts: a displaced sphere with the face count of the reference's yoga6 mesh, and a
5000-face torus."""
import torch


def displaced_sphere(n=562, seed=0):
    """UV sphere of n x n quads (2 n^2 triangles, 631 688 for n = 562), radius 1 + 0.05 * seeded smooth noise"""
    g = torch.Generator().manual_seed(seed)
    th = torch.linspace(0.02, 3.12, n + 1)
    ph = torch.arange(n) * (2 * torch.pi / n)
    T, P = torch.meshgrid(th, ph, indexing="ij")
    k = torch.randint(1, 8, (6, 3), generator=g).float()
    a = torch.rand(6, generator=g) - 0.5
    r = 1 + 0.05 * sum(a[i] * torch.sin(k[i, 0] * T + k[i, 1] * P + k[i, 2]) for i in range(6))
    verts = torch.stack([r * torch.sin(T) * torch.cos(P), r * torch.cos(T), r * torch.sin(T) * torch.sin(P)], -1)
    idx = torch.arange((n + 1) * n).view(n + 1, n)
    a0, a1 = idx[:-1], idx[:-1].roll(-1, 1)
    b0, b1 = idx[1:], idx[1:].roll(-1, 1)
    faces = torch.cat([torch.stack([a0, b0, b1], -1).reshape(-1, 3), torch.stack([a0, b1, a1], -1).reshape(-1, 3)])
    return verts.reshape(-1, 3).contiguous(), faces.contiguous()


def torus(R=0.6, r=0.25, nu=100, nv=25):
    """(R + r cos v) (cos u, ., sin u), r sin v: nu x nv quads, 2 nu nv = 5000 triangles"""
    u = torch.arange(nu, dtype=torch.float64) * (2 * torch.pi / nu)
    v = torch.arange(nv, dtype=torch.float64) * (2 * torch.pi / nv)
    U, Vv = torch.meshgrid(u, v, indexing="ij")
    verts = torch.stack([(R + r * Vv.cos()) * U.cos(), r * Vv.sin(), (R + r * Vv.cos()) * U.sin()], -1).reshape(-1, 3)
    i, j = torch.meshgrid(torch.arange(nu), torch.arange(nv), indexing="ij")
    idx = lambda a, b: (a % nu) * nv + (b % nv)
    faces = torch.cat([torch.stack([idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)], -1).reshape(-1, 3),
                       torch.stack([idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)], -1).reshape(-1, 3)])
    return verts.float(), faces
