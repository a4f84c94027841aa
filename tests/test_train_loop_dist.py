"""CPU tests of the training loop's multi-rank pieces (dss_b200.training.train, dss_b200.parallel): the choice between
the single-GPU loop and a rank of a torchrun job, the device refusal before the group is joined, dealing a batch's
views, the exit agreement and the replica guard over 2 gloo CPU processes.  Every process is started in its own session
and its process group is killed on a timeout, so a failing test leaves nothing running."""
import json
import os
import signal
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from dss_b200.training import train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT = 120

_WORKER = r'''
import json, sys, torch, torch.distributed as dist
sys.path.insert(0, %(root)r)
from dss_b200.parallel import agree_any, check_replicas, replicas_differ
rank, port, mode = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%%d" %% port, rank=rank, world_size=2)
out = {}
try:
    if mode == "exit":
        group = dist.new_group(backend="gloo")
        left = None
        for it in range(20):
            # only rank 1's clock runs out, from iteration 7 on
            if agree_any(rank == 1 and it >= 7, group):
                left = it
                break
        out["left_at"] = left
        out["quiet"] = agree_any(False, group)
    else:
        g = torch.Generator().manual_seed(5)
        a, b = torch.randn(100, 3, generator=g), torch.rand(7, 3, generator=g)
        out["same"] = replicas_differ([a, b])
        ulp = a.clone()
        if rank == 1:
            ulp[17, 2] = torch.nextafter(ulp[17, 2], torch.tensor(float("inf")))
        out["ulp"] = replicas_differ([ulp, b])
        zero = b.clone()
        zero[3, 1] = 0.0 if rank == 0 else -0.0
        out["signed_zero"] = replicas_differ([a, zero])
        try:
            check_replicas((("points", a), ("normals", zero)))
            out["raised"] = None
        except RuntimeError as e:
            out["raised"] = str(e)
        check_replicas((("points", a), ("normals", b)))
finally:
    dist.destroy_process_group()
print("RESULT " + json.dumps(out))
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _communicate(procs, timeout=TIMEOUT):
    """outputs of ``procs`` (each the leader of its own session); on a timeout every session is killed"""
    try:
        return [p.communicate(timeout=timeout)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                os.killpg(p.pid, signal.SIGKILL)
                p.wait()


def _two_workers(tmp_path, mode):
    w = tmp_path / "worker.py"
    w.write_text(_WORKER % {"root": ROOT})
    port = _free_port()
    procs = [subprocess.Popen([sys.executable, str(w), str(r), str(port), mode], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True, cwd=ROOT, start_new_session=True)
             for r in range(2)]
    outs = _communicate(procs)
    res = []
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o
        res.append(json.loads(next(line for line in o.splitlines() if line.startswith("RESULT "))[7:]))
    return res


def test_single_gpu_loop_without_world_size(monkeypatch):
    calls = []

    class Recorder:
        def __init__(self, cfg, *args, **kwargs):
            calls.append((args, kwargs))

        def run(self, exit_after, max_it):
            return 0

    monkeypatch.setattr(train, "Trainer", Recorder)
    monkeypatch.setattr(train, "load_config", lambda path: {})
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    for world in (None, "1"):
        if world is None:
            monkeypatch.delenv("WORLD_SIZE", raising=False)
        else:
            monkeypatch.setenv("WORLD_SIZE", world)
        calls.clear()
        assert train.main(["--config", "unused.yml", "--max-it", "1"]) == 0
        assert calls == [((), {})]                       # no device, no grad_sync: the graphed single-GPU loop
        assert not (torch.distributed.is_available() and torch.distributed.is_initialized())
    assert train.dist_env({}) is None and train.dist_env({"WORLD_SIZE": "1", "RANK": "0"}) is None
    assert train.dist_env({"WORLD_SIZE": "4", "RANK": "3", "LOCAL_RANK": "1", "LOCAL_WORLD_SIZE": "2"}) == \
        {"rank": 3, "world": 4, "local_rank": 1, "local_world": 2}


def test_rank_devices():
    with pytest.raises(RuntimeError, match="2 local ranks share 1 visible GPU"):
        train.rank_device("nccl", 0, 2, 1)
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        train.rank_device("gloo", 0, 2, 0)
    assert train.rank_device("nccl", 3, 4, 8) == torch.device("cuda", 3)
    assert [train.rank_device("gloo", r, 3, 2) for r in range(3)] == [torch.device("cuda", i) for i in (0, 1, 0)]


def test_nccl_with_more_local_ranks_than_gpus_is_refused_before_joining(tmp_path):
    # rank 1 of 2 with no rank 0 anywhere: joining the group would wait for rank 0's store until the timeout
    local_world = torch.cuda.device_count() + 1
    env = dict(os.environ, PYTHONPATH=ROOT, WORLD_SIZE="2", RANK="1", LOCAL_RANK="1",
               LOCAL_WORLD_SIZE=str(local_world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()))
    p = subprocess.Popen([sys.executable, "-m", "dss_b200.training.train", "--config", str(tmp_path / "none.yml"),
                          "--dist-backend", "nccl"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         cwd=ROOT, env=env, start_new_session=True)
    out = _communicate([p], timeout=60)[0]
    assert p.returncode != 0, out
    assert "RuntimeError" in out and ("visible GPU" in out or "needs a CUDA device" in out), out


def test_dealing_a_batch():
    g = np.random.default_rng(4)
    cams = g.standard_normal((16, 4, 4)).astype(np.float32)
    for idx in ([0, 5, 5, 9, 2, 2, 2, 15], [7, 3, 11], [4], list(range(16))):
        for G in (1, 2, 3, 4, 8):
            parts = train.deal_batch(cams, idx, G)
            assert len(parts) == G
            # every position of the batch on exactly one rank (repeats kept)
            assert sorted(v for part in parts for v in part) == sorted(idx)
            sizes = [len(part) for part in parts]
            assert max(sizes) - min(sizes) <= 1
            if len(idx) < G:
                assert sizes.count(0) == G - len(idx)
            # every rank deals alike: the same result from its own copies of the inputs
            assert train.deal_batch(cams.copy(), list(idx), G) == parts
    # views that cost the same wherever they repeat
    assert train.deal_batch(cams, [3, 3], 2) == [[3], [3]]


def test_exit_agreement_over_two_gloo_processes(tmp_path):
    res = _two_workers(tmp_path, "exit")
    assert [r["left_at"] for r in res] == [7, 7]
    assert [r["quiet"] for r in res] == [False, False]


def test_replica_guard_over_two_gloo_processes(tmp_path):
    res = _two_workers(tmp_path, "replicas")
    for r in res:
        assert r["same"] is False
        assert r["ulp"] is True
        assert r["signed_zero"] is True
        assert r["raised"] and "points, normals" in r["raised"]


def test_ground_truth_checks_without_loading(tmp_path):
    # the checks every rank runs at start, while only rank 0 loads the ground truth: the errors ground_truth_cloud
    # would raise, from the data's arrays and file names alone
    from dss_b200.utils.dataset import MVRData
    np.savez(tmp_path / "data_dict.npz", camera_mat=np.tile(np.eye(4, dtype=np.float32), (4, 1, 1)),
             points=np.zeros((10, 3), np.float32), normals=np.ones((10, 3), np.float32))
    data, d = MVRData(str(tmp_path)), str(tmp_path)
    with pytest.raises(ValueError, match="eval_sampling"):
        train.check_ground_truth(data, d, 8000, "meshlab")
    with pytest.raises(FileNotFoundError, match="mesh.obj"):
        train.check_ground_truth(data, d, 8000, "uniform")
    with pytest.raises(ValueError, match="mesh.obj"):
        train.check_ground_truth(data, d, 8000, "poisson_disk")
    for n in (0, 10):                                   # the stored cloud: no mesh needed
        for sampling in ("uniform", "poisson_disk"):
            train.check_ground_truth(data, d, n, sampling)
    (tmp_path / "mesh.obj").write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n")
    for sampling in ("uniform", "poisson_disk"):
        train.check_ground_truth(data, d, 8000, sampling)
