"""Time the splat-size K-NN (dss_knn_points) on the bench cloud, next to the reference's brute force on the CPU."""
import time, json
import numpy as np, torch
from timing import card, events_ms
import oracle
from dss_b200.frnn_grid import knn_points_packed
from tests.util import sphere_cloud
dev = torch.device("cuda:0")
res = {}
for P in (100_000, 1_000_000, 4_000_000):
    pts = sphere_cloud(P)[0].to(dev)
    f = torch.zeros(1, dtype=torch.int64, device=dev); n = torch.tensor([P], dtype=torch.int64, device=dev)
    knn = lambda: knn_points_packed(pts, f, n, 7, 0.2, return_idx=False)
    for _ in range(3): d = knn()[0]
    ms = events_ms(knn, 10)
    h = float((0.5 * d[:, 1:].max(1)[0]).mean().clamp(5e-5, 1e-3))
    res[P] = {"ms": ms, "Mqueries_per_s": P / ms / 1e3, "h": h}
sub = sphere_cloud(20000)[0].numpy()
t0 = time.perf_counter(); oracle.knn_brute(sub, np.zeros(1, np.int64), np.array([20000]), sub, np.zeros(1, np.int64), np.array([20000]), 7, 0.2)
res["cpu_bruteforce_20k"] = {"s": time.perf_counter() - t0, "threads": oracle.num_threads()}
gpu = card()
res["card"], res["power_limit"] = gpu["name"], gpu["power_limit"]
print(json.dumps(res))
