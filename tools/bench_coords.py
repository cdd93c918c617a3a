"""Cost of utils.coords' neighbour searches on the GPU (csrc/coords.cu).

  kernel  CUDA-event ms of each search kernel, averaged over --iters launches after a warm-up:
          the k-nearest query (nn = 4 and 16), the ball query's count and fill passes, the
          trajectory walk, and the DBSCAN root and label passes
  e2e     wall time from host arrays to host arrays (ending in a device synchronise), median of
          --iters calls: get_nn_distances(nn=4), compare_coordinates(d_max=3),
          find_coord_clusters(rmax=3), cluster_coord(eps=1, min_samples=10) and
          subimg_trajectories(window 16, rmax=3).get_all_trajectories()
Workloads: jittered square lattices of 8 px spacing (tests/golden/coords_cases.py) — a 1024²
frame of about 1.6·10⁴ atoms, a 100-frame movie of about 4·10³ atoms per frame, and a 2·10⁵-atom
lattice.  Prints the card's name and power limit, then one JSON line per measurement.

    python tools/bench_coords.py [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import coords_cases as cc  # noqa: E402
from atomai_b200 import ops  # noqa: E402
from atomai_b200.utils import coords, graphx  # noqa: E402


def _events(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _wall(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def kernels(tag, frames, iters):
    counts = [len(c) for c in frames.values()]
    pos = coords._xyz(np.concatenate([c[:, :2] for c in frames.values()]))
    F, N = len(frames), len(pos)
    t = {}
    for k in (5, 17):
        cl = coords._Cells(pos, counts, coords._knn_side(pos, F, k, np.inf))
        oidx = torch.empty(N, k, dtype=torch.int32, device="cuda")
        odist = torch.empty(N, k, dtype=torch.float64, device="cuda")
        t[f"knn_nn{k - 1}"] = _events(lambda: ops.coords_knn(
            cl.pos, cl.cells, cl.frame, cl.pos, cl.keys, cl.perm, cl.foff, cl.lo, cl.side, cl.dims,
            k, np.inf, oidx, odist), iters)
    span = float((pos.max(0) - pos.min(0)).max())
    cb = coords._Cells(pos, [N], coords._ball_side(3.0, span))
    q = cb.pos[:counts[0]]
    qc = cb.cells[:counts[0]]
    args = (q, qc, cb.pos, cb.keys, cb.perm, cb.lo, cb.side, cb.dims, 3.0)
    cnt = torch.empty(len(q), dtype=torch.int64, device="cuda")
    t["ball_count"] = _events(lambda: ops.coords_ball(*args, cnt=cnt), iters)
    rowptr = graphx._offsets(cnt)
    M = int(rowptr[-1])
    oi = torch.empty(max(M, 1), dtype=torch.int32, device="cuda")
    od = torch.empty(max(M, 1), dtype=torch.float64, device="cuda")
    t["ball_fill"] = _events(lambda: ops.coords_ball(*args, rowptr, oi, od), iters)
    cw = coords._Cells(pos, counts, coords._knn_side(pos, F, 1, 3.0))
    out = torch.empty(counts[0], F, 4, dtype=torch.int32, device="cuda")
    t["walk"] = _events(lambda: ops.coords_walk(
        cw.pos[:counts[0]], cw.cells[:counts[0]], cw.pos, cw.cells, cw.keys, cw.perm, cw.foff,
        cw.lo, cw.side, cw.dims, 3.0, 1024, 1024, 8, 16, out), iters)
    # DBSCAN passes over the bond search's eps-neighbourhoods (eps = 1)
    side = 1.0 * (1 + 2.0 ** -48 * (span + 1))
    lo = pos.min(0)
    dims = np.floor((pos.max(0) - lo) / side).astype(np.int64) + 1
    keys = torch.empty(N, dtype=torch.int64, device="cuda")
    ops.graph_cell_keys(cb.pos, None, lo, side, dims, keys)
    keys, perm = torch.sort(keys, stable=True)
    cut = torch.ones(1, 1, dtype=torch.float64, device="cuda")
    deg = torch.empty(N, dtype=torch.int32, device="cuda")
    bargs = (cb.pos, None, None, keys, perm, cut, lo, side, dims)
    ops.graph_bonds(*bargs, None, deg)
    rp = graphx._offsets(deg)
    cols = torch.empty(max(int(rp[-1]), 1), dtype=torch.int32, device="cuda")
    ops.graph_bonds(*bargs, rp, cols)
    parent = torch.empty(N, dtype=torch.int32, device="cuda")
    flag = torch.empty(1, dtype=torch.int32, device="cuda")
    t["dbscan_roots"] = _events(lambda: ops.coords_dbscan_roots(rp, cols, 10, parent, flag), iters)
    rank = torch.cumsum(parent == torch.arange(N, dtype=torch.int32, device="cuda"), 0) - 1
    labels = torch.empty(N, dtype=torch.int64, device="cuda")
    t["dbscan_labels"] = _events(lambda: ops.coords_dbscan_labels(rp, cols, parent, rank, labels),
                                 iters)
    print(json.dumps({"what": "kernel", "workload": tag, "frames": F, "atoms": N,
                      "ball_rows": M, "ms": {k: round(v, 4) for k, v in t.items()}}), flush=True)


def e2e(tag, frames, iters):
    first = frames[0]
    img = np.zeros((max(frames) + 1, 1024, 1024), np.float32)
    rng = np.random.default_rng(0)
    c2 = first.copy()
    c2[:, :2] += rng.normal(0, 0.8, (len(c2), 2))
    t = {"get_nn_distances": _wall(lambda: coords.get_nn_distances(frames, 4), iters),
         "compare_coordinates": _wall(lambda: coords.compare_coordinates(first, c2, 3.0), iters),
         "find_coord_clusters": _wall(lambda: coords.find_coord_clusters({0: first}, frames, 3),
                                      iters),
         "cluster_coord": _wall(lambda: coords.cluster_coord(frames, 1.0, 10), iters)}
    if len(frames) > 1:
        t["subimg_trajectories"] = _wall(lambda: coords.subimg_trajectories(
            img, frames, 16, 0, 3).get_all_trajectories(), iters)
    print(json.dumps({"what": "e2e", "workload": tag, "frames": len(frames),
                      "atoms": int(sum(len(c) for c in frames.values())),
                      "s": {k: round(v, 4) for k, v in t.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}", flush=True)
    work = {"frame_1024": {0: cc.lattice(127, 1, origin=4.0)},
            "movie_100x4k": cc.movie(100, 64, 2, drift=0.5),
            "lattice_200k": {0: cc.lattice(448, 3, origin=4.0)}}
    for tag, frames in work.items():
        kernels(tag, frames, a.iters)
        e2e(tag, frames, max(3, a.iters // 3))


if __name__ == "__main__":
    main()
