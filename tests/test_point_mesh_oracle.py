"""CPU: the float64 point-to-mesh oracle (tests/point_mesh_oracle.py) against closed forms -- the seven Voronoi regions
of a triangle, degenerate faces, a closed cube -- and against dense samples of every face."""
import numpy as np
import pytest
import torch

from tests.point_mesh_oracle import closest_points, point_mesh_distance

D = torch.float64


def t(*rows):
    return torch.tensor(rows, dtype=D)


@pytest.mark.parametrize("q, x", [
    ((-1.0, -1.0, 0.5), (0.0, 0.0, 0.0)),        # vertex a
    ((2.0, -0.5, 0.0), (1.0, 0.0, 0.0)),         # vertex b
    ((-0.5, 2.0, 0.3), (0.0, 1.0, 0.0)),         # vertex c
    ((0.5, -1.0, 0.2), (0.5, 0.0, 0.0)),         # edge ab
    ((-1.0, 0.5, 0.0), (0.0, 0.5, 0.0)),         # edge ac
    ((1.0, 1.0, 0.5), (0.5, 0.5, 0.0)),          # edge bc
    ((0.2, 0.3, 0.7), (0.2, 0.3, 0.0)),          # interior
])
def test_voronoi_regions(q, x):
    a, b, c = t(0, 0, 0), t(1, 0, 0), t(0, 1, 0)
    got = closest_points(t(*q), a, b, c)
    assert torch.allclose(got, t(*x), rtol=0, atol=1e-15)
    verts = torch.stack([a, b, c]).float()
    sq, face, cl, second = point_mesh_distance(t(*q)[None], verts, torch.tensor([[0, 1, 2]]))
    assert face.tolist() == [0] and second.tolist() == [float("inf")]
    assert abs(float(sq[0]) - float(((t(*q) - t(*x)) ** 2).sum())) <= 1e-15


@pytest.mark.parametrize("tri, q, x", [
    (((0, 0, 0), (1, 0, 0), (2, 0, 0)), (1.5, 1, 0), (1.5, 0, 0)),      # collinear: the long edge ca
    (((0, 0, 0), (1, 0, 0), (2, 0, 0)), (3, 0, 1), (2, 0, 0)),          # collinear, beyond an end
    (((0, 0, 0), (2, 0, 0), (1, 0, 0)), (-1, 0, 0), (0, 0, 0)),         # collinear, middle vertex last
    (((0, 0, 0), (0, 0, 0), (1, 0, 0)), (0.5, 1, 0), (0.5, 0, 0)),      # repeated vertex: a segment
    (((0, 0, 0), (1, 0, 0), (1, 0, 0)), (2, 3, 0), (1, 0, 0)),          # repeated vertex, beyond the end
    (((1, 2, 3), (1, 2, 3), (1, 2, 3)), (1, 2, 4), (1, 2, 3)),          # all three equal: a point
])
def test_degenerate_faces(tri, q, x):
    got = closest_points(t(*q), t(*tri[0]), t(*tri[1]), t(*tri[2]))
    assert torch.isfinite(got).all()
    assert torch.allclose(got, t(*x), rtol=0, atol=1e-15)


def cube_mesh():
    """the closed unit cube [0, 1]^3, 12 triangles"""
    v = torch.tensor([[i, j, k] for i in (0, 1) for j in (0, 1) for k in (0, 1)], dtype=torch.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = [tri for a, b, c, d in quads for tri in ((a, b, c), (a, c, d))]
    return v, torch.tensor(f)


def test_cube_inside_and_outside():
    v, f = cube_mesh()
    g = torch.Generator().manual_seed(0)
    q = (torch.rand(4000, 3, generator=g, dtype=D) * 3 - 1).float().double()
    sq, face, cl, _ = point_mesh_distance(q, v, f)
    r = (q - 0.5).abs()
    outside = (r - 0.5).clamp(min=0)
    exact = torch.where((r <= 0.5).all(1), (0.5 - r.max(1).values) ** 2, (outside ** 2).sum(1))
    assert ((q > 0) & (q < 1)).all(1).any() and (~((q >= 0) & (q <= 1)).all(1)).any()
    assert torch.allclose(sq, exact, rtol=1e-12, atol=1e-15)
    # the closest point lies on the surface, at the reported distance
    assert torch.allclose(((q - cl) ** 2).sum(1), sq, rtol=1e-12, atol=1e-15)
    assert ((cl >= -1e-15) & (cl <= 1 + 1e-15)).all()
    assert (face >= 0).all() and (face < 12).all()


def test_never_above_dense_samples():
    g = torch.Generator().manual_seed(1)
    tris = torch.rand(40, 3, 3, generator=g) * 2 - 1
    tris[0, 2] = tris[0, 1]                                   # repeated vertex
    tris[1, 2] = 2 * tris[1, 1] - tris[1, 0]                  # collinear
    tris[2, 1] = tris[2, 0] + torch.tensor([1e-3, 0, 0])      # sliver
    tris[2, 2] = tris[2, 0] + torch.tensor([0.9, 1e-4, 0])
    verts = tris.reshape(-1, 3)
    faces = torch.arange(120).reshape(40, 3)
    q = (torch.rand(300, 3, generator=g) * 4 - 2).double()
    sq, face, cl, _ = point_mesh_distance(q, verts, faces)
    n = 40
    u, w = torch.meshgrid(torch.arange(n + 1, dtype=D) / n, torch.arange(n + 1, dtype=D) / n, indexing="ij")
    keep = (u + w) <= 1
    u, w = u[keep], w[keep]
    tv = tris.double()
    samples = (tv[:, None, 0] * (1 - u - w)[None, :, None] + tv[:, None, 1] * u[None, :, None]
               + tv[:, None, 2] * w[None, :, None]).reshape(-1, 3)
    dmin = torch.cdist(q, samples).pow(2).min(1).values
    assert (sq <= dmin + 1e-12).all()
    # and not below the true distance: the closest point is on the reported face
    a, b, c = tv[face, 0], tv[face, 1], tv[face, 2]
    assert torch.equal(closest_points(q, a, b, c), cl)


def test_ties_unusable_faces_and_queries():
    v = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [float("nan"), 0, 0]], dtype=torch.float32)
    f = torch.tensor([[0, 1, 3], [0, 1, 2], [2, 1, 0], [0, 1, 7]])
    q = torch.tensor([[0.2, 0.2, 1.0], [float("inf"), 0, 0]], dtype=D)
    sq, face, cl, second = point_mesh_distance(q, v, f)
    assert face.tolist() == [1, -1]                # faces 1 and 2 tie exactly: the smaller index
    assert float(sq[0]) == 1.0 and float(second[0]) == 1.0
    assert np.isnan(float(sq[1])) and torch.isnan(cl[1]).all()
    sq, face, _, _ = point_mesh_distance(q, v, f[[0, 3]])
    assert torch.isnan(sq).all() and face.tolist() == [-1, -1]
