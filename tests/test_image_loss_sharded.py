"""CPU test of the view-sharded image loss: ``image_loss_torch(..., group=...)`` over 2 gloo processes, each holding
some of the views, against ``image_loss_torch`` over all the views in float64 -- the loss values and every rank's slice
of the RGBA gradient."""
import os
import socket
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_WORKER = r'''
import sys, torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
from dss_b200.training.losses import image_loss_torch
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%(port)d", rank=int(sys.argv[1]), world_size=2)
rank = dist.get_rank()
N, H, W = 5, 11, 13
g = torch.Generator().manual_seed(3)
rgba0 = torch.rand(N, H, W, 4, generator=g, dtype=torch.float64)
rgba0[..., 3] = torch.where(torch.rand(N, H, W, generator=g) < 0.3, 0.0, rgba0[..., 3])
img = torch.rand(N, H, W, 3, generator=g, dtype=torch.float64)
mask = torch.where(torch.rand(N, H, W, generator=g) < 0.4, 0.0, torch.rand(N, H, W, generator=g, dtype=torch.float64))
# views 3 and 4 see no pixel where both masks are non-zero: the rank that holds only them has M = 0
rgba0[3:, ..., 3] = torch.where(mask[3:] != 0, 0.0, rgba0[3:, ..., 3])
SPLITS = {"M=0 on rank 1": ([0, 1, 2], [3, 4]), "2+3": ([1, 3], [0, 2, 4]), "5+0": ([0, 1, 2, 3, 4], []),
          "uint8": ([4], [0, 1, 2, 3])}
for name, parts in SPLITS.items():
    m = (mask != 0).to(torch.uint8) if name == "uint8" else mask
    for lams in ((1.0, 1.0), (0.7, 2.5), (0.0, 1.0), (1.0, 0.0)):
        full = rgba0.clone().requires_grad_(True)
        want = image_loss_torch(full, img, m, *lams)
        want["loss"].backward()
        mine = parts[rank]
        part = rgba0[mine].clone().requires_grad_(True)
        got = image_loss_torch(part, img[mine], m[mine], *lams, group=dist.group.WORLD)
        got["loss"].backward()
        for k in ("loss", "loss_dr_rgb", "loss_dr_silhouette"):
            w, v = float(want[k]), float(got[k])
            assert abs(v - w) <= 1e-13 * abs(w) + 1e-300, (name, lams, k, v, w)
        scale = float(full.grad.abs().max())
        assert part.grad.shape == (len(mine), H, W, 4)
        err = float((part.grad - full.grad[mine]).abs().max()) if mine else 0.0
        assert err <= 1e-13 * scale, (name, lams, err, scale)
        if name == "M=0 on rank 1" and rank == 1:
            assert not (m[mine].bool() & part.detach()[..., 3].bool()).any() and not part.grad[..., :3].any()
dist.destroy_process_group()
print("rank", rank, "ok")
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def test_sharded_image_loss_torch_equals_the_loss_over_all_views():
    with tempfile.TemporaryDirectory() as d:
        w = os.path.join(d, "worker.py")
        with open(w, "w") as f:
            f.write(_WORKER % {"root": ROOT, "port": _free_port()})
        procs = [subprocess.Popen([sys.executable, w, str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                  text=True) for r in range(2)]
        try:
            outs = [p.communicate(timeout=180)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and "rank %d ok" % r in o, o
