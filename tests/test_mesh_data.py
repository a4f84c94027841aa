"""CPU: the mesh rasterizer's rules on hand-built cases (tests/mesh_oracle.py), mesh files, the data helpers of
dss_b200.utils.create_mvr_data and the data directory it writes, read back by MVRData."""
import math
import os
import random

import numpy as np
import pytest
import torch

from tests.mesh_oracle import pix_to_ndc, rasterize_mesh_naive

# ---- meshes shared with the GPU tests ------------------------------------------------------------------------------


def icosphere(subdiv):
    """unit icosphere: (verts (V,3) f32, faces (F,3) int64)"""
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    verts = [np.asarray(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(subdiv):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = verts[a] + verts[b]
                verts.append(p / np.linalg.norm(p))
                mid[k] = len(verts) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return torch.tensor(np.asarray(verts), dtype=torch.float32), torch.tensor(f, dtype=torch.int64)


def torus(R=0.6, r=0.25, nu=48, nv=24):
    u, v = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    verts = np.stack([(R + r * np.cos(v)) * np.cos(u), r * np.sin(v), (R + r * np.cos(v)) * np.sin(u)], -1).reshape(-1, 3)
    idx = lambda i, j: (i % nu) * nv + (j % nv)
    faces = []
    for i in range(nu):
        for j in range(nv):
            faces += [(idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)), (idx(i, j), idx(i + 1, j + 1), idx(i, j + 1))]
    return torch.tensor(verts, dtype=torch.float32), torch.tensor(faces, dtype=torch.int64)


# ---- hand-built cases: screen-space vertices (identity cameras), S, and the check ---------------------------------

def at(a, S, xi, yi):
    """value of pixel-index (xi, yi) in an (S,S) image (row S-1-yi, column S-1-xi)"""
    return a[S - 1 - yi, S - 1 - xi]


def _shared_edge():
    # two faces meeting on y = -0.125, the centres of pixel row 3 at S = 8: that row is covered by neither
    v = [(-1, -0.125, 1), (1, -0.125, 1), (0, 1, 1), (0, -1, 1)]
    f = [(0, 1, 2), (0, 3, 1)]

    def check(p2f, z):
        assert pix_to_ndc(3, 8) == np.float32(-0.125)
        assert all(at(p2f, 8, x, 3) == -1 for x in range(8))
        assert at(p2f, 8, 4, 4) == 0 and at(p2f, 8, 4, 2) == 1
    return v, f, 8, check


def _vertex_on_centre(flip=False):
    v = [(0.125, 0.125, 1), (0.9, 0.2, 1), (0.2, 0.9, 1)]
    f = [(0, 2, 1)] if flip else [(0, 1, 2)]

    def check(p2f, z):
        assert at(p2f, 8, 4, 4) == -1        # the centre on v0: w1 = w2 = 0
        assert at(p2f, 8, 5, 5) == 0 and at(z, 8, 5, 5) == np.float32(1)
    return v, f, 8, check


def _area(scale):
    # a sliver through the centre of S = 3 with |E(v0, v1, v2)| = 4h: skipped at or below 1e-8
    h = np.float32(scale * 1e-8 / 4)
    v = [(-1, -h, 1), (1, -h, 1), (0, h, 1)]

    def check(p2f, z):
        if scale < 1:
            assert (p2f == -1).all()
        else:
            hh = float(h)
            den = -4 * hh + 1e-8                  # the +1e-8 of the barycentric denominator dominates
            assert at(p2f, 3, 1, 1) == 0
            assert at(z, 3, 1, 1) == pytest.approx(-4 * hh / den, rel=1e-3)
            assert (p2f >= 0).sum() == 1
    return v, [(0, 1, 2)], 3, check


def _straddle(behind=False):
    zs = (-1.0, -1.0, -0.5) if behind else (-1.0, -1.0, 2.0)
    v = [(-3, -3, zs[0]), (3, -3, zs[1]), (0, 4, zs[2])]

    def check(p2f, z):
        if behind:
            assert (p2f == -1).all()
            return
        for yi in range(8):
            yc = float(pix_to_ndc(yi, 8))
            pz = -1 + 3 * (yc + 3) / 7          # depth along y; >= 0 from y = -2/3 on
            for xi in range(8):
                assert at(p2f, 8, xi, yi) == (0 if pz >= 0 else -1)
                if pz >= 0:
                    assert at(z, 8, xi, yi) == pytest.approx(pz, abs=1e-5)
    return v, [(0, 1, 2)], 8, check


def _zero_depth(sign):
    zz = math.copysign(0.0, sign)
    v = [(-3, -3, zz), (3, -3, zz), (0, 4, zz)]

    def check(p2f, z):
        assert (p2f == 0).all() and (z == 0).all()
    return v, [(0, 1, 2)], 4, check


def _ties():
    v = [(-3, -3, 1), (3, -3, 1), (0, 4, 1)]

    def check(p2f, z):
        assert (p2f == 0).all() and np.allclose(z, 1, rtol=0, atol=1e-6)
    return v, [(0, 1, 2), (0, 1, 2), (0, 1, 2)], 4, check   # the same values: exact ties


def _nonfinite():
    nan, inf = float("nan"), float("inf")
    v = [(nan, 0, 1), (1, 0, 1), (0, 1, 1), (inf, 0, 1), (-1, -1, 1), (1, -1, 1), (0, 0, nan), (-inf, 1, 1),
         (0, inf, 1), (0.5, 0.5, inf)]
    f = [(0, 1, 2), (3, 4, 5), (6, 5, 4), (7, 4, 5), (8, 4, 5), (9, 4, 5)]

    def check(p2f, z):
        # NaN or infinite x, y and a NaN z cover nothing; a vertex at z = +inf with finite x, y follows the rules like
        # any other: its face covers where its barycentrics are positive, at depth +inf
        assert set(np.unique(p2f)) == {-1, 5}
        assert (z[p2f == 5] == np.inf).all()
    return v, f, 8, check


def _s1():
    v = [(-0.5, -0.5, 2), (0.5, -0.5, 2), (0, 0.5, 2)]

    def check(p2f, z):
        assert p2f.shape == (1, 1) and p2f[0, 0] == 0 and z[0, 0] == pytest.approx(2, abs=1e-6)
    return v, [(0, 1, 2)], 1, check


HAND_CASES = {"shared_edge": _shared_edge, "vertex_on_centre": _vertex_on_centre,
              "mirrored_winding": lambda: _vertex_on_centre(flip=True), "area_above": lambda: _area(1.05),
              "area_below": lambda: _area(0.95), "straddles_z0": _straddle, "behind": lambda: _straddle(True),
              "depth_plus_zero": lambda: _zero_depth(1.0), "depth_minus_zero": lambda: _zero_depth(-1.0),
              "ties": _ties, "nonfinite": _nonfinite, "s1": _s1}


@pytest.mark.parametrize("case", sorted(HAND_CASES))
def test_oracle_hand_built_cases(case):
    v, f, S, check = HAND_CASES[case]()
    p2f, z = rasterize_mesh_naive(np.asarray(v, np.float32)[None], np.asarray(f), S)
    check(p2f[0], z[0])


def test_oracle_depth_order_and_views():
    # two faces over the whole image, the farther one first: the nearer wins; a second view swaps the depths
    v = np.array([[(-3, -3, 2), (3, -3, 2), (0, 4, 2), (-3, -3, 1), (3, -3, 1), (0, 4, 1)],
                  [(-3, -3, 1), (3, -3, 1), (0, 4, 1), (-3, -3, 2), (3, -3, 2), (0, 4, 2)]], np.float32)
    p2f, z = rasterize_mesh_naive(v, [(0, 1, 2), (3, 4, 5)], 5)
    assert (p2f[0] == 1).all() and (p2f[1] == 0).all() and np.allclose(z, 1, rtol=0, atol=1e-6)


# ---- mesh files --------------------------------------------------------------------------------------------------

def _write_ply(path, verts, polys, fmt, count_t="uchar", index_t="int", extra_face_prop=False):
    from dss_b200.utils.io import _PLY_TYPES
    end = {"binary_little_endian": "<", "binary_big_endian": ">"}.get(fmt)
    head = ["ply", "format %s 1.0" % fmt, "comment test", "element vertex %d" % len(verts),
            "property float x", "property float y", "property float z", "element face %d" % len(polys)]
    if extra_face_prop:
        head.append("property uchar flags")
    head += ["property list %s %s vertex_indices" % (count_t, index_t), "end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        if end is None:
            for v in verts:
                f.write(("%r %r %r\n" % tuple(float(x) for x in v)).encode())
            for p in polys:
                f.write((("7 " if extra_face_prop else "") + " ".join(str(x) for x in [len(p)] + list(p)) + "\n").encode())
        else:
            f.write(np.asarray(verts, end + "f4").tobytes())
            for p in polys:
                if extra_face_prop:
                    f.write(np.asarray([7], "u1").tobytes())
                f.write(np.asarray([len(p)], end + _PLY_TYPES[count_t]).tobytes())
                f.write(np.asarray(p, end + _PLY_TYPES[index_t]).tobytes())


def _fan_expect(polys):
    return np.asarray([(p[0], p[i], p[i + 1]) for p in polys for i in range(1, len(p) - 1)], np.int64)


VERTS = np.random.default_rng(0).normal(size=(7, 3)).astype(np.float32)


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
@pytest.mark.parametrize("count_t,index_t", [("uchar", "int"), ("int", "uint"), ("uint8", "short")])
@pytest.mark.parametrize("polys", [[(0, 1, 2), (2, 3, 4)], [(0, 1, 2, 3), (3, 4, 5, 6)], [(0, 1, 2), (1, 2, 3, 4, 5)]])
def test_read_mesh_ply(tmp_path, fmt, count_t, index_t, polys):
    from dss_b200.utils.io import read_mesh
    path = str(tmp_path / "m.ply")
    _write_ply(path, VERTS, polys, fmt, count_t, index_t, extra_face_prop=len(polys[1]) == 5)
    v, f = read_mesh(path)
    assert v.dtype == np.float32 and f.dtype == np.int64
    np.testing.assert_array_equal(v, VERTS)
    np.testing.assert_array_equal(f, _fan_expect(polys))


def test_read_mesh_obj_forms_and_save_obj_round_trip(tmp_path):
    from dss_b200.utils.io import read_mesh, save_obj
    path = tmp_path / "m.obj"
    lines = ["# comment", "o thing"] + ["v %.9g %.9g %.9g" % tuple(v) for v in VERTS[:4]] + ["vt 0 0", "vn 0 0 1"]
    lines += ["f 1 2 3", "f 1/1 3/1 4/1", "f 2/1/1 3/1/1 4/1/1", "f 1//1 2//1 4//1", "f -4 -3 -2"]
    lines += ["v %.9g %.9g %.9g" % tuple(v) for v in VERTS[4:]] + ["f 4 5 6 7", "f -1 -2 -3"]
    path.write_text("\n".join(lines) + "\n")
    v, f = read_mesh(str(path))
    np.testing.assert_array_equal(v, VERTS)
    np.testing.assert_array_equal(f, [(0, 1, 2), (0, 2, 3), (1, 2, 3), (0, 1, 3), (0, 1, 2), (3, 4, 5), (3, 5, 6),
                                      (6, 5, 4)])
    out = str(tmp_path / "sub" / "out.obj")
    save_obj(out, v, f)
    v2, f2 = read_mesh(out)
    np.testing.assert_array_equal(v2, v)
    np.testing.assert_array_equal(f2, f)


@pytest.mark.parametrize("text", ["v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf -4 1 2\n",
                                  "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 0 1 2\n"])
def test_read_mesh_obj_bad_index_raises(tmp_path, text):
    from dss_b200.utils.io import read_mesh
    p = tmp_path / "bad.obj"
    p.write_text(text)
    with pytest.raises(ValueError):
        read_mesh(str(p))


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
def test_read_mesh_ply_bad_index_raises(tmp_path, fmt):
    from dss_b200.utils.io import read_mesh
    path = str(tmp_path / "bad.ply")
    _write_ply(path, VERTS, [(0, 1, 7)], fmt)
    with pytest.raises(ValueError):
        read_mesh(path)


def test_reference_yoga6_reads():
    path = "/root/reference/example_data/mesh/yoga6.ply"
    if not os.path.exists(path):
        pytest.skip("the reference's example mesh is not present")
    from dss_b200.utils.io import read_mesh
    v, f = read_mesh(path)
    assert v.shape == (315808, 3) and f.shape == (631628, 3)
    assert f.min() >= 0 and f.max() < len(v)


# ---- helpers -----------------------------------------------------------------------------------------------------

def test_camera_sampler_ranges_order_and_seed():
    from dss_b200.core.camera import CameraSampler, FoVPerspectiveCameras
    mk = lambda seed: CameraSampler(50, 8, distance_range=((1.2, 2.2),), camera_type=FoVPerspectiveCameras,
                                    camera_params={"znear": 0.1}, generator=torch.Generator().manual_seed(seed))
    s = mk(1)
    assert ((s.distances >= 1.2) & (s.distances <= 2.2)).all() and (s.distances[:-1] >= s.distances[1:]).all()
    assert ((s.azim >= -180) & (s.azim < 180)).all() and ((s.elev >= -90) & (s.elev < 90)).all()
    assert (s.at.abs() <= 0.05).all()
    batches = list(s)
    assert [len(c) for c in batches] == [8] * 6 + [2] and batches[0].znear == pytest.approx(0.1)
    centres = torch.cat([c.get_camera_center() for c in batches])
    np.testing.assert_allclose((centres - s.at).norm(dim=1).numpy(), s.distances.numpy(), rtol=1e-5)
    assert torch.equal(mk(1).R, s.R) and not torch.equal(mk(2).R, s.R)


def _cam(seed):
    from tests.util import random_cameras
    return random_cameras(1, seed)


@pytest.mark.parametrize("point_lights", [False, True])
@pytest.mark.parametrize("has_specular", [False, True])
def test_tri_color_lights_formula(point_lights, has_specular):
    from dss_b200.utils.create_mvr_data import get_tri_color_lights_for_view
    cam = _cam(3)
    l = get_tri_color_lights_for_view(cam, has_specular=has_specular, point_lights=point_lights,
                                      generator=torch.Generator().manual_seed(5))
    # float64 restatement: directions in the frame z = normalize(cross(C, u)), x = normalize(cross(C, z)), y = z x x
    C = cam.get_camera_center().double()[0]
    u = torch.rand(1, 3, generator=torch.Generator().manual_seed(5)).double()[0]
    z = torch.nn.functional.normalize(torch.cross(C, u, dim=0), dim=0)
    x = torch.nn.functional.normalize(torch.cross(C, z, dim=0), dim=0)
    y = torch.cross(z, x, dim=0)
    e, a = math.radians(30), torch.tensor([-60.0, 60.0, 180.0], dtype=torch.float64) * math.pi / 180
    local = torch.stack([math.cos(e) * torch.sin(a), torch.full_like(a, math.sin(e)), math.cos(e) * torch.cos(a)], 1)
    want = local @ torch.stack([x, y, z])
    got = l._vec[0].double() / (5 if point_lights else 1)
    np.testing.assert_allclose(got.numpy(), want.numpy(), atol=1e-5)
    dif = np.array([[0, 0, 0.8], [0, 0.8, 0], [0.8, 0, 0]])
    np.testing.assert_allclose(l.diffuse_color[0].numpy(), dif * (0.85 if has_specular else 1), atol=1e-7)
    np.testing.assert_allclose(l.specular_color[0].numpy(), dif * (0.15 if has_specular else 0), atol=1e-7)
    np.testing.assert_allclose(l.ambient_color[0].numpy(), [[0.2, 0.2, 0.2]], atol=1e-7)
    assert type(l).__name__ == ("PointLights" if point_lights else "DirectionalLights")


@pytest.mark.parametrize("point_lights", [False, True])
def test_single_light_formula_maps_the_direction_as_a_point(point_lights):
    from dss_b200.utils.create_mvr_data import get_light_for_view
    cam = _cam(4)
    l = get_light_for_view(cam, point_lights=point_lights, has_specular=True, rng=random.Random(7))
    r = random.Random(7)
    e, a = math.radians(r.randint(10, 90)), math.radians(r.randint(0, 360))
    d = np.array([math.cos(e) * math.sin(a), math.sin(e), math.cos(e) * math.cos(a)])
    M = cam.get_world_to_view_transform().get_matrix()[0].double().numpy()
    want = (np.append(d, 1.0) @ np.linalg.inv(M))[:3]             # (d 1) inv(M): the translation is applied
    got = l._vec[0, 0].double().numpy() / (5 if point_lights else 1)
    np.testing.assert_allclose(got, want, atol=1e-5)
    assert np.linalg.norm(want - d @ np.linalg.inv(M)[:3, :3]) > 0.1   # the quirk is visible
    np.testing.assert_allclose(l.diffuse_color[0, 0].numpy(), [0.17] * 3, atol=1e-7)
    np.testing.assert_allclose(l.specular_color[0, 0].numpy(), [0.03] * 3, atol=1e-7)
    np.testing.assert_allclose(l.ambient_color[0, 0].numpy(), [0.6] * 3, atol=1e-7)


def test_surface_sampler_in_face_normals_and_area_frequency():
    from scipy import stats
    from dss_b200.utils.create_mvr_data import sample_points_from_mesh
    verts, faces = icosphere(1)
    g = torch.Generator().manual_seed(0)
    verts = verts * (1 + 0.5 * torch.rand(verts.shape[0], 1, generator=g))      # faces of unequal areas
    n = 50000
    p, nrm = sample_points_from_mesh(verts, faces, n, generator=torch.Generator().manual_seed(1))
    # the faces that hold each sample: plane distance <= 1e-6 and barycentrics in [0, 1] (two only on an edge)
    tri = verts[faces].double()
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    fn = torch.nn.functional.normalize(torch.cross(e1, e2, dim=1), dim=1)
    q = p.double()[:, None, :] - tri[None, :, 0]                                     # (n, F, 3)
    dist = (q * fn[None]).sum(-1).abs()
    d00, d01, d11 = (e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)
    d20, d21 = (q * e1[None]).sum(-1), (q * e2[None]).sum(-1)
    den = d00 * d11 - d01 * d01
    w1, w2 = (d11 * d20 - d01 * d21) / den, (d00 * d21 - d01 * d20) / den
    w0 = 1 - w1 - w2
    tol = 1e-5
    holds = (dist <= 1e-6) & (w0 >= -tol) & (w1 >= -tol) & (w2 >= -tol)
    assert bool(holds.any(1).all())
    same_normal = (nrm.double()[:, None, :] - fn[None]).abs().amax(-1) <= 1e-6
    assert bool((holds & same_normal).any(1).all())
    fidx = holds.int().argmax(1)
    area = torch.cross(e1, e2, dim=1).norm(dim=1) / 2
    expect = (area / area.sum() * n).numpy()
    counts = np.bincount(fidx.numpy(), minlength=len(faces))
    chi2 = ((counts - expect) ** 2 / expect).sum()
    assert stats.chi2.sf(chi2, len(faces) - 1) > 1e-3, chi2


def test_writer_directory_reads_back_through_mvrdata(tmp_path):
    from dss_b200.core.lighting import PointLights
    from dss_b200.utils.create_mvr_data import light_value_dict, write_mvr_data
    from dss_b200.utils.dataset import MVRData
    from dss_b200.utils.io import read_mesh
    from tests.util import random_cameras
    N, S = 3, 16
    rng = np.random.default_rng(0)
    images = rng.uniform(-0.2, 1.3, (N, S, S, 4)).astype(np.float32)
    masks = rng.random((N, S, S)) > 0.5
    cams = random_cameras(N, 2)
    cam_mat = cams.get_world_to_view_transform().get_matrix().numpy()
    lights = [light_value_dict(PointLights(ambient_color=rng.random((1, 1, 3)), diffuse_color=rng.random((1, 3, 3)),
                                           specular_color=rng.random((1, 3, 3)), location=rng.normal(size=(1, 3, 3))))
              for _ in range(N)]
    verts, faces = icosphere(1)
    pts, nrm = rng.normal(size=(50, 3)).astype(np.float32), rng.normal(size=(50, 3)).astype(np.float32)
    out = write_mvr_data(str(tmp_path / "d"), verts.numpy(), faces.numpy(), images, masks, cam_mat, lights, pts, nrm,
                         True, {"znear": 0.1})
    data = MVRData(out)
    assert len(data) == N
    for i in range(N):
        want = (np.clip(images[i], 0, 1) * np.float32(255)).astype(np.uint8)
        np.testing.assert_array_equal(np.round(data.images[i].numpy().transpose(1, 2, 0) * 255).astype(np.uint8),
                                      want[..., :3])
        np.testing.assert_array_equal(data.masks[i][0].numpy().astype(bool), masks[i])
        np.testing.assert_array_equal(data[i]["camera_mat"], cam_mat[i])
    items = [data[i] for i in range(N)]
    L = PointLights(**{k: torch.stack([torch.as_tensor(it["lights"][k]) for it in items]) for k in items[0]["lights"]})
    for k, t in (("ambient_color", L.ambient_color), ("diffuse_color", L.diffuse_color),
                 ("specular_color", L.specular_color), ("location", L.location)):
        np.testing.assert_array_equal(t.numpy(), np.concatenate([d[k] for d in lights]).astype(np.float32))
    cloud = data.get_pointclouds()
    np.testing.assert_array_equal(cloud.points_packed().numpy(), pts)
    np.testing.assert_array_equal(cloud.normals_packed().numpy(), nrm)
    got = data.get_cameras()
    assert got.znear == pytest.approx(0.1)
    np.testing.assert_array_equal(got.R.numpy(), cams.R.numpy())
    np.testing.assert_array_equal(got.T.numpy(), cams.T.numpy())
    v, f = read_mesh(os.path.join(out, "mesh.obj"))
    np.testing.assert_array_equal(v, verts.numpy())
    np.testing.assert_array_equal(f, faces.numpy())
    dd = np.load(os.path.join(out, "data_dict.npz"), allow_pickle=True)
    assert str(dd["lights_type"]) == "DSS.core.lighting.PointLights"
    assert str(dd["cameras_type"]) == "pytorch3d.renderer.cameras.FoVPerspectiveCameras"
    np.testing.assert_array_equal(dd["colors"], np.ones((50, 3), np.float32))
