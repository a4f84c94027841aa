"""The shading-gradient bound of tests/shading_grad_oracle.py on the CPU: a float32 restatement of the kernels'
expression order meets it on every family, the same restatement at 17 significant bits (128 times coarser) breaks it
on every output (the bound is not vacuous), the float64 values equal float64 torch autograd of the lighting formula
away from the eps boundary, and at the boundary (|x| = float32(1e-6) exactly, one ulp either side) they follow float32
torch autograd through F.normalize: the gradient passes through the norm at equality."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dss_b200.core import lighting
from tests.shading_grad_oracle import Bounded, edge_slots, ordinary_slots, rounded, slot_outputs, within

CASES = [(kind, L, shin) for kind in ("sun", "point") for L, shin in ((1, 1.0), (2, 13.5), (8, 64.0))]
OUTPUTS = ("alb", "nrm", "pos", "cam", "amb", "vec", "cd", "cs")


def _families(kind, L, shin):
    return {"edges": edge_slots(kind, L, shin, seed=L)[0], "ordinary": ordinary_slots(3000, kind, L, shin, seed=L)}


def _ratios(s, bits):
    want = slot_outputs(Bounded, s)
    got = slot_outputs(rounded(bits), s)
    res = {}
    for k in OUTPUTS:
        r, same = within(got[k], *want[k])
        assert same.all(), k
        res[k] = float(r.max())
    return res


@pytest.mark.parametrize("kind,L,shin", CASES)
def test_float32_restatement_meets_the_bound(kind, L, shin):
    for fam, s in _families(kind, L, shin).items():
        r = _ratios(s, 24)
        print("%s L=%d shin=%g %s: worst ratio %s" % (kind, L, shin, fam, {k: "%.3g" % v for k, v in r.items()}))
        assert max(r.values()) <= 1, (fam, r)


@pytest.mark.parametrize("kind,L,shin", CASES)
def test_bound_is_not_vacuous_at_17_bits(kind, L, shin):
    for fam, s in _families(kind, L, shin).items():
        r = _ratios(s, 17)
        print("%s L=%d shin=%g %s at 17 bits: %s" % (kind, L, shin, fam, {k: "%.3g" % v for k, v in r.items()}))
        for k, v in r.items():
            assert v > 1, (fam, k, v)


def _torch_grads(s, dtype, eps=1e-6):
    """autograd of the lighting formula (dss_b200/core/lighting.py: F.normalize(eps=1e-6)) per slot in `dtype`
    -> dict of the oracle's outputs"""
    t = {k: torch.tensor(np.asarray(s[k]), dtype=dtype, requires_grad=k != "gc") for k in
         ("p", "n", "alb", "cam", "lights", "amb", "gc")}
    rows = t["lights"]
    vec = rows[..., 0:3] - t["p"][:, None] if s["light_type"] else rows[..., 0:3]
    dif = lighting.diffuse(t["n"], rows[..., 3:6], vec)
    spe = lighting.specular(t["p"], t["n"], vec, rows[..., 6:9], t["cam"], s["shin"])
    col = t["alb"] * (t["amb"] + dif) + spe
    g = torch.autograd.grad(col, [t[k] for k in ("alb", "n", "p", "cam", "amb", "lights")], t["gc"])
    out = dict(alb=g[0], nrm=g[1], pos=g[2], cam=g[3], amb=g[4], vec=g[5][..., 0:3], cd=g[5][..., 3:6],
               cs=g[5][..., 6:9])
    return {k: v.double().numpy() for k, v in out.items()}


_AT_EPS = ("eps", "at camera", "at light", "zero normal")


@pytest.mark.parametrize("kind,L,shin", CASES)
def test_float64_values_equal_torch_autograd_away_from_eps(kind, L, shin):
    for fam, s in _families(kind, L, shin).items():
        want = _torch_grads(s, torch.float64)
        got = slot_outputs(Bounded, s)
        keep = np.ones(len(s["p"]), bool)
        if fam == "edges":
            labels = edge_slots(kind, L, shin, seed=L)[1]
            keep = np.array([not any(a in lab for a in _AT_EPS) for lab in labels])
        for k in OUTPUTS:
            w, g = want[k][keep], got[k][0][keep]
            np.testing.assert_allclose(g, w, rtol=1e-9, atol=1e-12 * max(np.abs(w).max(), 1.0), err_msg=(fam, k))


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_exact_eps_follows_float32_torch_autograd(kind):
    """|n|, |c - p| and |l - p| at float32(1e-6) exactly and one ulp either side: float32 F.normalize passes the
    gradient through the norm at equality (the projected gradient), the linear branch holds only below it; the two
    differ by O(1), far outside the bound"""
    s, labels = edge_slots(kind, 2, 13.5, seed=5)
    rows = [i for i, lab in enumerate(labels) if "eps" in lab or lab in ("at camera", "at light", "zero normal")]
    s = dict(s, **{k: s[k][rows] for k in ("p", "n", "alb", "cam", "lights", "amb", "gc")})
    want = slot_outputs(Bounded, s)
    got = _torch_grads(s, torch.float32)
    for k in OUTPUTS:
        r, same = within(got[k], *want[k], safety=4.0)   # torch's own float32 order: a few times the kernels' count
        assert same.all() and (r <= 1).all(), (kind, k, float(r.max()))
    # the branch matters there: at |n| = eps exactly the projected and the linear gradients differ
    i = rows.index(labels.index("|n|=eps"))
    n = torch.tensor(s["n"][i:i + 1], dtype=torch.float32, requires_grad=True)
    gy = torch.tensor([[0.3, 0.7, -0.2]])
    (gn,) = torch.autograd.grad(F.normalize(n, p=2, dim=-1, eps=1e-6), n, gy)
    assert float(s["n"][i, 2]) == float(np.float32(1e-6)) and float(gn[0, 2]) == 0.0   # along z: projected out
    assert abs(float(want["nrm"][0][i, 2])) < 1e-3 * np.abs(want["nrm"][0][i]).max()
