"""K nearest neighbours within a radius (SURVEY.md section 8(f) row 1).

CPU: the oracle's brute force against golden vectors minted from the reference's own ground truth FRNNBruteForceCPU
(tests/golden/make_golden_knn.py) and against the compiled witness's outputs (tests/golden/ref_cpu_witness.npz).
GPU: the grid kernel (through the C ABI) against the oracle, bit for bit -- distances AND indices, ties included --
plus size-independent properties at 1M points."""
import os

import numpy as np
import pytest
import torch

import oracle
from tests.util import golden_case

REF_CPU_GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_cpu_witness.npz")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "knn_frnn_bruteforce.npz")
CASES = [("k7_r0.2", 7, 0.2), ("k12_r0.05", 12, 0.05)]


def _clouds(d):
    return sorted(k[:-len("__points")] for k in d.files if k.endswith("__points") and not k.startswith("edge_"))


def test_oracle_knn_reproduces_reference_bruteforce_golden_vectors():
    d = np.load(GOLD)
    assert len(_clouds(d)) >= 4
    for name in _clouds(d):
        p = d[name + "__points"]
        f, n = np.zeros(1, np.int64), np.array([len(p)], np.int64)
        for tag, K, r in CASES:
            dist, idx = oracle.knn_brute(p, f, n, p, f, n, K, r)
            assert np.array_equal(dist, d["%s__%s__dists" % (name, tag)]), (name, tag)   # same sums, same order: bit-exact
            assert np.array_equal(idx, d["%s__%s__idxs" % (name, tag)]), (name, tag)     # ties resolved like the reference
    # the small radius leaves some lists short (-1 padding exercised), the self match is always first
    short = d["teapot_normal_dense__k12_r0.05__idxs"]
    assert (short[:, -1] == -1).any() and (short[:, 0] == np.arange(len(short))).all()
    # the edge families, padded batches (tests/golden/make_golden_knn.py: edge_families)
    names = [c[0] for c in edge_cases(d)]
    assert {"edge_duplicates", "edge_r2_boundary", "edge_lattice_ties", "edge_nonfinite", "edge_long_line",
            "edge_ragged"} <= set(names)
    for name, pts, lens, K, r in edge_cases(d):
        first = np.arange(len(lens), dtype=np.int64) * pts.shape[1]
        dist, idx = oracle.knn_brute(pts.reshape(-1, 3), first, lens, pts.reshape(-1, 3), first, lens, K, r)
        dist, idx = dist.reshape(pts.shape[:2] + (K,)), idx.reshape(pts.shape[:2] + (K,))
        assert np.array_equal(dist.view(np.uint32), d[name + "__dists"].view(np.uint32)), name
        assert np.array_equal(idx, d[name + "__idxs"]), name
    # what the families are there for, in the reference's own output
    nf = d["edge_nonfinite__points"][0]
    bad = ~np.isfinite(nf).all(1)
    assert bad.sum() == 6 and (d["edge_nonfinite__idxs"][0][bad] == -1).all()
    on = d["edge_r2_boundary__idxs"][0]
    assert (on[:20, 1] == -1).all() and (on[40:60, 1] == np.arange(60, 80)).all()    # at r: out; one ulp inside: in
    z = (d["edge_duplicates__dists"][0] == 0).all(1)                          # 13 copies of 3 points, K = 8
    assert z.sum() == 39 and (np.diff(d["edge_duplicates__idxs"][0][z], axis=1) > 0).all()


def edge_cases(d):
    """-> [(name, points (N,P,3), lengths (N,), K, r)] of the edge families stored in the K-NN golden file"""
    names = sorted(k[:-len("__lengths")] for k in d.files if k.startswith("edge_") and k.endswith("__lengths"))
    return [(n, d[n + "__points"], d[n + "__lengths"], int(d[n + "__K"]), float(d[n + "__r"])) for n in names]


def _witness_clouds():
    rng = np.random.default_rng(3)
    p1 = rng.uniform(-1, 1, (2, 300, 3)).astype(np.float32)      # queries != points, two clouds of different length
    p2 = rng.uniform(-1, 1, (2, 400, 3)).astype(np.float32)
    l1, l2 = np.array([300, 180], np.int64), np.array([400, 250], np.int64)
    return p1, p2, l1, l2


def witness_frnn_bruteforce_cpu(ref):
    """the reference's FRNNBruteForceCPU (oracle/_ref/dss_ref_frnn_cpu) on the clouds of the test below"""
    p1, p2, l1, l2 = _witness_clouds()
    idxs, dists = ref.frnn_bf_cpu(torch.from_numpy(p1), torch.from_numpy(p2), torch.from_numpy(l1), torch.from_numpy(l2),
                                  5, 0.4)
    return dict(idxs=idxs.numpy(), dists=dists.numpy())


def test_oracle_knn_matches_compiled_reference_witness():
    want = golden_case(REF_CPU_GOLDEN, "frnn_bf")
    idxs, dists = want["idxs"], want["dists"]
    p1, p2, l1, l2 = _witness_clouds()
    q = np.concatenate([p1[0, :300], p1[1, :180]])
    pts = np.concatenate([p2[0, :400], p2[1, :250]])
    dist, idx = oracle.knn_brute(q, np.array([0, 300]), l1, pts, np.array([0, 400]), l2, 5, 0.4)
    assert np.array_equal(dist[:300], dists[0, :300]) and np.array_equal(dist[300:], dists[1, :180])
    assert np.array_equal(idx[:300], idxs[0, :300]) and np.array_equal(idx[300:], idxs[1, :180])


def test_cell_model_puts_a_close_pair_two_cells_apart():
    """Why the ring bound's slack grows with the grid.  On a line longer than 1024 r the radius clamp sets the cell to
    r and the grid to up to 2^21 cells along x; the computed cell coordinate t = fl(fl(x - gmin) * inv_cell) is then
    known to ~0.1 cell only, so a fixed slack of 1e-3 cells is unsound.  This float32 model of the kernel's grid puts
    x = 130105.83f and 130106.02f, 0.977 cells apart, two cells apart; tests/test_gpu_knn_edges.py runs the kernel on
    a cloud of such pairs (tests.util.knn_long_line)."""
    from tests.util import knn_cell_model, knn_long_line
    f32 = np.float32
    gmin = f32(-1234.567)
    ends = np.array([[gmin, 0, 0], [f32(gmin + f32(419000)), 0, 0]], f32)
    lo, cell, inv, res, cell_of = knn_cell_model(ends, 0.2)
    assert cell == f32(0.2) and inv == f32(5) and res[0] == 2095001 and (1 << 20) < res[0] <= (1 << 21)
    a, b = f32(130105.83), f32(130106.02)
    ca, cb = cell_of(np.array([[a, 0, 0], [b, 0, 0]], f32))[:, 0]
    assert cb - ca == 2
    d = f32(b - a)
    assert float(d) == 0.1953125 and float(d) / float(cell) < 0.999
    reach2 = f32(f32(f32(f32(1) - f32(1e-3)) * cell) ** 2)       # the old stop test after ring 1
    assert f32(d * d) < reach2
    # the slack the kernel derives (16 u (maxres + 2)) covers the error of t at this size: 2 err < slack
    t_exact = (np.float64(b) - np.float64(gmin)) * np.float64(inv)
    t_comp = np.float64(f32(f32(b - gmin) * inv))
    slack = (res.max() + 2) * 2.0 ** -20
    assert abs(t_comp - t_exact) > 1e-3 and 2 * 2.0001 * 2.0 ** -24 * (res.max() + 1) < slack
    # the generator of the GPU family: every triple as documented, on the grid of the whole cloud
    pts, A, B, C = knn_long_line()
    assert len(A) >= 60
    _, cell2, _, res2, cell_of2 = knn_cell_model(pts, 0.2)
    assert cell2 == cell and (res2 == [2095001, 1, 1]).all()
    ca, cb, cc = cell_of2(pts[A]), cell_of2(pts[B]), cell_of2(pts[C])
    assert (cb[:, 0] - ca[:, 0] == 2).all() and (cc == ca).all()
    dab = ((pts[B] - pts[A]).astype(f32) ** 2).astype(f32).sum(1, dtype=f32)
    dac = ((pts[C] - pts[A]).astype(f32) ** 2).astype(f32).sum(1, dtype=f32)
    assert (dab < dac).all() and (dac < reach2).all()


def test_cell_model_grid_fits_for_adversarial_extents():
    """The argument in knn_params_kernel: for any finite extents and any radius, 1 <= res[k] and prod res <= 2^21
    (on the float32 model; the GPU file runs the kernel on such clouds)."""
    from tests.util import knn_cell_model
    f32 = np.float32
    big = f32(3e38)
    cases = [([[-big, 0, 0], [big, 0, 0]], r) for r in (-1.0, 0.2, 1e-30)]
    cases += [([[0, 0, 0], [1e8, 0, 0], [0, 1e8, 0], [0, 0, 1e8]], r) for r in (-1.0, 0.2, 1e-6)]
    cases += [([[-big, -big, -big], [big, big, big]], r) for r in (-1.0, 0.2)]
    cases += [([[0, 0, 0], [1e-30, 1e-30, 1e-30]], r) for r in (-1.0, 0.2)]
    cases += [([[0, 0, 0]], 0.2), ([[-0.0, 0, 0], [0.0, 0, 0]], -1.0)]
    for p, r in cases:
        _, cell, inv, res, _ = knn_cell_model(np.array(p, f32), r)
        assert np.isfinite(cell) and cell > 0 and (res >= 1).all() and int(np.prod(res)) <= (1 << 21), (p, r, res)


# ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_knn_kernel_matches_golden_and_oracle(cuda_device):
    from dss_b200.frnn_grid import knn_points_packed
    d = np.load(GOLD)
    for name in _clouds(d):
        p = torch.from_numpy(d[name + "__points"]).to(cuda_device)
        f = torch.zeros(1, dtype=torch.int64, device=cuda_device)
        n = torch.tensor([p.shape[0]], dtype=torch.int64, device=cuda_device)
        for tag, K, r in CASES:
            dist, idx = knn_points_packed(p, f, n, K, r)
            assert np.array_equal(dist.cpu().numpy(), d["%s__%s__dists" % (name, tag)]), (name, tag)
            assert np.array_equal(idx.cpu().numpy(), d["%s__%s__idxs" % (name, tag)]), (name, tag)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,P,K,r", [("sphere", 20000, 7, 0.2), ("cube", 15000, 16, 0.1), ("line", 5000, 7, -1.0),
                                        ("tiny", 5, 7, 0.2), ("clustered", 12000, 32, 0.3)])
def test_knn_kernel_matches_oracle_ragged_batches(cuda_device, kind, P, K, r):
    from dss_b200.frnn_grid import knn_points_packed
    rng = np.random.default_rng(len(kind) + P)
    if kind == "sphere":
        x = rng.standard_normal((P, 3)); x = 0.5 * x / np.linalg.norm(x, axis=1, keepdims=True)
    elif kind == "cube":
        x = rng.uniform(-0.5, 0.5, (P, 3))
    elif kind == "line":
        x = np.stack([np.linspace(-1, 1, P), np.zeros(P), np.zeros(P)], 1) + rng.standard_normal((P, 3)) * 1e-4
    elif kind == "tiny":
        x = rng.uniform(-0.1, 0.1, (P, 3))
    else:
        c = rng.uniform(-1, 1, (20, 3))
        x = c[rng.integers(0, 20, P)] + rng.standard_normal((P, 3)) * 0.02
    x = x.astype(np.float32)
    # three clouds of different lengths packed back to back (one of them empty)
    cuts = [0, P // 3, P // 3, P]
    first = np.array(cuts[:-1], np.int64)
    num = np.array([cuts[i + 1] - cuts[i] for i in range(3)], np.int64)
    want_d, want_i = oracle.knn_brute(x, first, num, x, first, num, K, r)
    t = lambda a: torch.from_numpy(a).to(cuda_device)
    got_d, got_i = knn_points_packed(t(x), t(first), t(num), K, r)
    assert np.array_equal(got_d.cpu().numpy(), want_d)
    assert np.array_equal(got_i.cpu().numpy(), want_i)
    # separate query set (general mode), including queries outside the bounding box of the points
    q = (x[::7] * 1.3 + 0.01).astype(np.float32)
    a = min(10, len(q))
    qfirst = np.array([0, a, a], np.int64)
    qnum = np.array([a, 0, len(q) - a], np.int64)
    want_d, want_i = oracle.knn_brute(q, qfirst, qnum, x, first, num, K, r)
    got_d, got_i = knn_points_packed(t(x), t(first), t(num), K, r, t(q), t(qfirst), t(qnum))
    assert np.array_equal(got_d.cpu().numpy(), want_d)
    assert np.array_equal(got_i.cpu().numpy(), want_i)


@pytest.mark.gpu
def test_frnn_grid_points_signature_and_h_rule(cuda_device):
    """the reference-facing twin (padded batches, int64 idxs, -1 padding) and the splat-size rule built on it
    (rasterizer.py:313-326)."""
    from dss_b200.frnn_grid import frnn_grid_points
    rng = np.random.default_rng(1)
    N, P = 2, 3000
    pts = torch.from_numpy(rng.uniform(-0.5, 0.5, (N, P, 3)).astype(np.float32)).to(cuda_device)
    lens = torch.tensor([P, 1800], dtype=torch.int64, device=cuda_device)
    dists, idxs, nn, grid = frnn_grid_points(pts, pts, lens, lens, K=7, r=0.2, return_nn=True)
    assert dists.shape == (N, P, 7) and idxs.dtype == torch.int64 and nn.shape == (N, P, 7, 3) and grid is None
    assert (dists[1, 1800:] == -1).all() and (idxs[1, 1800:] == -1).all()
    x = pts.cpu().numpy()
    for n in range(N):
        L = int(lens[n])
        wd, wi = oracle.knn_brute(x[n, :L], np.zeros(1, np.int64), np.array([L]), x[n, :L], np.zeros(1, np.int64),
                                  np.array([L]), 7, 0.2)
        assert np.array_equal(dists[n, :L].cpu().numpy(), wd) and np.array_equal(idxs[n, :L].cpu().numpy(), wi)
    # pytorch3d-style twin (no radius, zero padding)
    from dss_b200.frnn_grid import knn_points
    kd, ki, _ = knn_points(pts, pts, lens, lens, K=12)
    wd, wi = oracle.knn_brute(x[1, :1800], np.zeros(1, np.int64), np.array([1800]), x[1, :1800], np.zeros(1, np.int64),
                              np.array([1800]), 12, -1.0)
    assert np.array_equal(kd[1, :1800].cpu().numpy(), wd) and np.array_equal(ki[1, :1800].cpu().numpy(), wi)
    assert (kd[1, 1800:] == 0).all() and (ki[1, 1800:] == 0).all()
    ok = idxs[0] >= 0
    g = torch.gather(pts[0][None].expand(P, -1, -1), 1, idxs[0].clamp(min=0)[..., None].expand(-1, -1, 3))
    assert torch.equal(nn[0][ok], g[ok])


@pytest.mark.gpu
def test_knn_fullsize_properties(cuda_device):
    """1M points (BASELINE headline cloud): self match first, ascending, inside the radius, and exact agreement with a
    brute-force torch search for a random sample of queries."""
    from dss_b200.frnn_grid import knn_points_packed
    from tests.util import sphere_cloud
    P, K, r = 1_000_000, 7, 0.2
    pts = sphere_cloud(P)[0].to(cuda_device)
    f = torch.zeros(1, dtype=torch.int64, device=cuda_device)
    n = torch.tensor([P], dtype=torch.int64, device=cuda_device)
    d, i = knn_points_packed(pts, f, n, K, r)
    assert (i[:, 0] == torch.arange(P, device=cuda_device)).all() and (d[:, 0] == 0).all()
    assert (d[:, 1:] >= d[:, :-1]).all() and (d >= 0).all() and (d < r * r).all()
    sel = torch.randperm(P, generator=torch.Generator().manual_seed(0))[:512].to(cuda_device)
    diff = pts[sel][:, None, :] - pts[None, :, :]
    d2 = (diff[..., 0] * diff[..., 0] + diff[..., 1] * diff[..., 1]) + diff[..., 2] * diff[..., 2]
    want = torch.topk(d2, K, dim=1, largest=False)[0]
    assert torch.equal(want, d[sel])
