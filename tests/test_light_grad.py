"""Per-view lights and light gradients, host side: pack_lights / make_shading layouts, broadcasting and errors, the
gradient from the packed rows back to the light tensors, the float64 closed form that dss_light_backward evaluates
against autograd through the torch shading, the entry point's argument checks (no device needed), and lights built
from MVRData items the way the reference trainer builds them."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dss_b200 import _lib, ops
from dss_b200.core.lighting import DirectionalLights, PointLights, pack_lights
from dss_b200.core.texture import apply_lighting, camera_centres
from dss_b200.ops import Shading, make_shading
from dss_b200.utils.dataset import MVRData
from tests.util import scene


def _per_view(kind, N=3, L=2, seed=0):
    """lights with a direction / location per view (N,L,3), colours shared (1,L,3), ambient per view (N,1,3)"""
    g = torch.Generator().manual_seed(seed)
    vec = torch.randn(N, L, 3, generator=g)
    kw = dict(ambient_color=0.2 * torch.rand(N, 1, 3, generator=g), diffuse_color=0.5 * torch.rand(1, L, 3, generator=g),
              specular_color=0.3 * torch.rand(1, L, 3, generator=g))
    if kind == "sun":
        return DirectionalLights(direction=vec, **kw)
    return PointLights(location=2.0 * vec, **kw)


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_pack_lights_per_view_shapes_and_broadcasting(kind):
    N, L = 3, 2
    lights = _per_view(kind, N, L)
    rows, amb, k = pack_lights(lights)
    assert rows.shape == (N, L, 9) and amb.shape == (N, 3) and k == lights.kind
    for n in range(N):
        torch.testing.assert_close(rows[n, :, 0:3], lights._vec[n], rtol=0, atol=0)
        torch.testing.assert_close(rows[n, :, 3:6], lights.diffuse_color[0], rtol=0, atol=0)   # batch 1 broadcast
        torch.testing.assert_close(rows[n, :, 6:9], lights.specular_color[0], rtol=0, atol=0)
        torch.testing.assert_close(amb[n], lights.ambient_color[n].sum(0), rtol=0, atol=0)
    # ambient colours of several lights are summed per view, shared ones broadcast
    two = DirectionalLights(ambient_color=torch.tensor([[[0.1, 0.2, 0.3], [0.05, 0.0, 0.1]]]),
                            diffuse_color=torch.rand(1, 2, 3), specular_color=torch.rand(1, 2, 3),
                            direction=torch.randn(N, 2, 3))
    _, amb2, _ = pack_lights(two)
    torch.testing.assert_close(amb2, torch.tensor([[0.15, 0.2, 0.4]]).expand(N, 3))


def test_pack_lights_of_one_set_is_unchanged():
    lights = DirectionalLights(ambient_color=(((0.3, 0.25, 0.2), (0.1, 0.1, 0.15)),),
                               diffuse_color=(((0.6, 0.5, 0.4), (0.2, 0.3, 0.5)),),
                               specular_color=(((0.5, 0.5, 0.4), (0.3, 0.2, 0.6)),),
                               direction=(((0.3, 1.0, 0.4), (-0.8, 0.1, 0.5)),))
    rows, amb, k = pack_lights(lights)
    want = torch.cat([lights.direction[0], lights.diffuse_color[0], lights.specular_color[0]], 1)
    assert rows.shape == (2, 9) and amb.shape == (3,) and k == 0
    assert torch.equal(rows, want) and torch.equal(amb, lights.ambient_color[0].sum(0))


def test_bad_light_batches_raise():
    bad = DirectionalLights(direction=torch.randn(2, 1, 3), diffuse_color=torch.rand(3, 1, 3))
    with pytest.raises(ValueError, match="batch 1 or N"):
        pack_lights(bad)
    view = scene(10, 3, seed=0)[4]
    with pytest.raises(ValueError, match="batch 1 or N"):
        make_shading(_per_view("sun", N=4), view)
    sh = make_shading(_per_view("sun", N=3), view)
    assert sh.lights.shape == (3, 2, 9) and sh.ambient.shape == (3, 3)
    assert make_shading(DirectionalLights(), view).lights.shape == (1, 9)
    # the render operator checks the layouts against N before it looks at the device
    cam = camera_centres(view)
    for lights, amb, msg in ((sh.lights, sh.ambient[0], "shading.ambient"), (sh.lights[:2], sh.ambient[:2], "shading.lights"),
                             (sh.lights[0], sh.ambient, "shading.ambient"), (torch.zeros(3, 9, 9), sh.ambient, "shading.lights")):
        with pytest.raises(RuntimeError, match=msg):
            ops._check_shading(Shading(lights, amb, cam), 3, None)


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_gradient_flows_from_packed_rows_to_the_light_tensors(kind):
    N, L = 3, 2
    lights = _per_view(kind, N, L)
    leaves = {name: getattr(lights, name).requires_grad_() for name in ("_vec", "diffuse_color", "specular_color",
                                                                       "ambient_color")}
    rows, amb, _ = pack_lights(lights)
    g = torch.Generator().manual_seed(3)
    Wr, Wa = torch.randn(N, L, 9, generator=g), torch.randn(N, 3, generator=g)
    ((rows * Wr).sum() + (amb * Wa).sum()).backward()
    torch.testing.assert_close(leaves["_vec"].grad, Wr[..., 0:3])
    torch.testing.assert_close(leaves["diffuse_color"].grad, Wr[..., 3:6].sum(0, keepdim=True))       # broadcast: summed
    torch.testing.assert_close(leaves["specular_color"].grad, Wr[..., 6:9].sum(0, keepdim=True))
    torch.testing.assert_close(leaves["ambient_color"].grad, Wa[:, None, :])
    # make_shading keeps the rows differentiable (device move included)
    lights._vec.grad = None
    sh = make_shading(lights, scene(10, N, seed=0)[4])
    sh.lights[..., 0:3].sum().backward()
    torch.testing.assert_close(lights._vec.grad, torch.ones(N, L, 3))


def light_grads64(p, nrm, alb, rows, kind, cam, gc, shininess):
    """float64 closed form of dss_light_backward for one view: p, nrm, alb, gc (P,3), rows (L,9), cam (3,) ->
    (grad_rows (L,9), grad_ambient (3,)), the per-light formulas of csrc/render.cu"""
    nh = F.normalize(nrm, dim=-1, eps=1e-6)[:, None, :]
    v = F.normalize(cam - p, dim=-1, eps=1e-6)[:, None, :]
    vec, cd, cs = rows[None, :, 0:3], rows[None, :, 3:6], rows[None, :, 6:9]
    draw = vec - p[:, None, :] if kind else vec.expand(p.shape[0], -1, -1)
    dlen = draw.norm(dim=-1, keepdim=True).clamp(min=1e-6)
    d = draw / dlen
    cos = (nh * d).sum(-1, keepdim=True)
    lam = cos.clamp(min=0)
    r = -d + 2 * cos * nh
    alpha = (v * r).sum(-1, keepdim=True).clamp(min=0) * (cos > 0)
    pw = torch.where(alpha > 0, alpha.pow(shininess), torch.zeros_like(alpha))
    ga = (gc * alb)[:, None, :]
    g_alpha = torch.where(alpha > 0, (gc[:, None, :] * cs).sum(-1, keepdim=True) * shininess
                          * alpha.pow(shininess - 1), torch.zeros_like(alpha))
    g_r = v * g_alpha
    g_cos = torch.where(cos > 0, (ga * cd).sum(-1, keepdim=True), torch.zeros_like(cos)) + 2 * (g_r * nh).sum(-1, keepdim=True)
    g_d = nh * g_cos - g_r
    g_vec = (g_d - d * (d * g_d).sum(-1, keepdim=True)) / dlen
    g_rows = torch.cat([g_vec, ga * lam, gc[:, None, :] * pw], -1).sum(0)
    return g_rows, (gc * alb).sum(0)


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_closed_form_equals_autograd_through_the_torch_shading_float64(kind):
    N, P0, shin = 3, 300, 13.5
    pts, nrm, col, _, view, _ = scene(P0, N, seed=9)
    nrm = nrm * 0.9
    lights = _per_view(kind, N, 2, seed=4)
    lights._vec[1, 0] = -lights._vec[1, 0]                # a light behind part of the surface
    p, n, a = pts.double(), nrm.double(), col.double()
    cam = camera_centres(view.double())
    idx = torch.arange(N).repeat_interleave(P0)
    gc = torch.randn(N * P0, 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    gc[torch.rand(N * P0, generator=torch.Generator().manual_seed(2)) < 0.5] = 0      # invisible slots
    # autograd w.r.t. the packed rows: the same shading rebuilt from rows that are leaves
    rows, ambient, _ = pack_lights(lights)
    rows, ambient = rows.detach().double().requires_grad_(), ambient.detach().double().requires_grad_()
    lk = (DirectionalLights if kind == "sun" else PointLights)(device="cpu")
    lk._vec, lk.diffuse_color, lk.specular_color = rows[..., 0:3], rows[..., 3:6], rows[..., 6:9]
    lk.ambient_color = ambient[:, None, :]
    amb, dif, spe = apply_lighting(p.repeat(N, 1), n.repeat(N, 1), lk, cam[idx], shininess=shin, view_idx=idx)
    g_rows, g_amb = torch.autograd.grad(((a.repeat(N, 1) * (amb + dif) + spe) * gc).sum(), (rows, ambient))
    for v in range(N):
        s = slice(v * P0, (v + 1) * P0)
        want_rows, want_amb = light_grads64(p, n, a, rows[v].detach(), lights.kind, cam[v], gc[s], shin)
        torch.testing.assert_close(g_rows[v], want_rows, rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(g_amb[v], want_amb, rtol=1e-10, atol=1e-12)
    assert g_rows[..., 0:3].abs().max() > 0 and g_rows[..., 6:9].abs().max() > 0


def _args(**kw):
    a = _lib.RenderArgs()
    fake = C.c_void_p(256)          # never dereferenced: every case fails an argument check first
    for f in ("points_world", "normals_world", "albedo", "lights", "ambient", "cam_centres", "grad_colours"):
        setattr(a, f, fake)
    a.n_views, a.shared_cloud, a.P0, a.P, a.image_size, a.points_per_pixel = 2, 1, 10, 20, 16, 5
    a.shade, a.n_lights = 1, 2
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_light_backward_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    out = C.c_void_p(512)
    null = C.c_void_p(0)

    def call(a, gl=out, ga=out):
        rc = lib.dss_light_backward(null, None if a is None else C.byref(a), gl, ga, null)
        return rc, _lib.last_error()

    cases = [
        (None, {}, "args is null"),
        (_args(shade=0), {}, "shade"),
        (_args(grad_colours=null), {}, "grad_colours"),
        (_args(points_world=null), {}, "points_world"),
        (_args(lights=null), {}, "shading needs"),
        (_args(n_lights=9), {}, "n_lights"),
        (_args(lights_per_view=2), {}, "lights_per_view must be 0 or 1"),
        (_args(lights_per_view=-1), {}, "lights_per_view must be 0 or 1"),
        (_args(lights_per_view=1, shade=0), {}, "lights_per_view needs"),
        (_args(P=21), {}, "P != n_views * P0"),
        (_args(lights_per_view=1), {"gl": null}, "ctx is null"),   # consistent arguments: only the missing context is left
        (_args(), {"ga": null}, "ctx is null"),
    ]
    for a, kw, msg in cases:
        rc, err = call(a, **kw)
        assert rc == -1 and msg in err, (msg, rc, err)
    # the forward refuses per-view lights without the shading as well
    rc = lib.dss_render_forward(null, C.byref(_args(lights_per_view=1, shade=0)), null)
    assert rc == -1


@pytest.mark.parametrize("kind", ["sun", "point"])
def test_lights_of_mvr_data_items_pack_per_view(tmp_path, kind):
    """scripts/create_mvr_data_from_mesh.py stores one light per image as lights_%d ((1,L,3) properties); the
    reference trainer stacks the items' `lights` dicts of a batch and builds one lights object from them
    (DSS/training/trainer.py:268-271)"""
    V = 4
    rng = np.random.default_rng(0)
    cam = np.tile(np.eye(4, dtype=np.float32), (V, 1, 1))
    cam[:, 3, 2] = 2.0
    vec_key = "direction" if kind == "sun" else "location"
    per_image = {}
    for i in range(V):
        per_image["lights_%d" % i] = np.array({
            "ambient_color": [[[0.6, 0.6, 0.6]]], "diffuse_color": [[[0.17, 0.17, 0.17]]],
            "specular_color": [[[0.03, 0.03, 0.03]]], vec_key: rng.standard_normal((1, 1, 3)).tolist()}, dtype=object)
    np.savez(tmp_path / "data_dict.npz", camera_mat=cam, points=rng.random((10, 3)), normals=rng.random((10, 3)),
             **per_image)
    data = MVRData(str(tmp_path))
    items = [data[i] for i in (2, 0, 3)]
    batch = {k: torch.stack([torch.as_tensor(it["lights"][k]) for it in items]) for k in items[0]["lights"]}
    lights = (DirectionalLights if kind == "sun" else PointLights)(**batch)
    rows, amb, k = pack_lights(lights)
    assert rows.shape == (3, 1, 9) and amb.shape == (3, 3) and k == lights.kind
    for j, i in enumerate((2, 0, 3)):
        want = np.asarray(per_image["lights_%d" % i].item()[vec_key], dtype=np.float32)[0, 0]
        np.testing.assert_array_equal(rows[j, 0, 0:3].numpy(), want)
    np.testing.assert_allclose(amb.numpy(), 0.6, rtol=1e-6)
    sh = make_shading(lights, torch.as_tensor(np.stack([it["camera_mat"] for it in items])))
    assert sh.lights.shape == (3, 1, 9) and sh.cam_centres.shape == (3, 3)
