"""Cost of utils.graphx on the GPU (csrc/graph.cu).

  kernel  per lattice: CUDA-event ms of each pass (bond count + fill with the cell-key sort, hop
          table, ring count + fill, shortest-path filter), averaged over --iters launches after a
          warm-up, with the ring count and the number of depth-first search steps of the count
          pass (the pruning by hop distance is what keeps the steps near the ring atoms)
  e2e     wall time (ending in a device synchronise) of find_cycles(c, [5, 6, 7]),
          find_cycle_clusters(c, [5, 7, 8]) and filter_subgraphs(c), median of --iters calls,
          and of filter_subgraphs over a 100-frame movie of 4·10³-atom frames (one batch)
Workloads: seeded honeycombs (tests/golden/graph_cases.py) with Stone–Wales defects, an amorphous
patch and stray atoms, at about 1.6·10⁴, 5·10⁴ and 2·10⁵ atoms.  Prints the card's name and power
limit, then one JSON line per measurement.

    python tools/bench_graph.py [--iters 10]
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

import graph_cases as gc  # noqa: E402
from atomai_b200 import ops  # noqa: E402
from atomai_b200.utils import graphx  # noqa: E402

LATTICES = {"16k": (62, 64, 12, 12.0), "50k": (110, 113, 30, 20.0), "200k": (220, 226, 100, 40.0)}


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


def kernels(tag, c, iters, max_depth=8):
    s = c.copy()
    s[:, :-1] *= gc.PX2ANG
    b = graphx._Bonds([s], gc.MAP_DICT, 1.2)
    N = b.N
    t = {"bonds": _events(lambda: graphx._Bonds([s], gc.MAP_DICT, 1.2), iters)}
    R = max_depth // 2
    t["hops"] = _events(lambda: (setattr(b, "ball", None), b.hop_table(R)), iters)
    bptr, ball = b.hop_table(R)
    cnt = torch.empty(N, 3, dtype=torch.int64, device="cuda")
    t["rings_count"] = _events(lambda: ops.graph_rings(b.rowptr, b.cols, bptr, ball, max_depth,
                                                       cnt=cnt), iters)
    rb, ab = graphx._offsets(cnt[:, 0]), graphx._offsets(cnt[:, 1])
    nr, na = int(rb[-1]), int(ab[-1])
    lens = torch.empty(nr, dtype=torch.int32, device="cuda")
    atoms = torch.empty(na, dtype=torch.int32, device="cuda")
    t["rings_fill"] = _events(lambda: ops.graph_rings(b.rowptr, b.cols, bptr, ball, max_depth,
                                                      rb[:-1], ab[:-1], lens, atoms), iters)
    off = graphx._offsets(lens)[:-1]
    keep = torch.empty(nr, dtype=torch.uint8, device="cuda")
    t["filter"] = _events(lambda: ops.graph_ring_filter(off, lens, atoms, bptr, ball, keep), iters)
    print(json.dumps({"what": "kernel", "lattice": tag, "atoms": N, "bonds": int(b.rowptr[-1]) // 2,
                      "max_depth": max_depth, "hop_entries": int(bptr[-1]), "rings": nr,
                      "kept": int(keep.sum()), "dfs_steps": int(cnt[:, 2].sum()),
                      "ms": {k: round(v, 4) for k, v in t.items()}}), flush=True)


def e2e(tag, c, iters):
    t = {"find_cycles_567": _wall(lambda: graphx.find_cycles(c, [5, 6, 7], gc.MAP_DICT, gc.PX2ANG), iters),
         "find_cycle_clusters_578": _wall(lambda: graphx.find_cycle_clusters(c, [5, 7, 8], gc.MAP_DICT,
                                                                             gc.PX2ANG), iters),
         "filter_subgraphs": _wall(lambda: graphx.filter_subgraphs(c, gc.MAP_DICT, gc.PX2ANG), iters)}
    print(json.dumps({"what": "e2e", "lattice": tag, "atoms": len(c),
                      "s": {k: round(v, 4) for k, v in t.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}", flush=True)
    for tag, (nx_, ny, sw, patch) in LATTICES.items():
        c = gc.honeycomb(nx_, ny, 1, n_sw=sw, patch=patch)
        c[:, :2] /= gc.PX2ANG
        kernels(tag, c, a.iters)
        e2e(tag, c, max(3, a.iters // 3))
    movie = {}
    for f in range(100):
        c = gc.honeycomb(31, 32, 100 + f, n_sw=4, patch=6.0, n_stray=5)
        c[:, :2] /= gc.PX2ANG
        movie[f] = c
    n = sum(len(c) for c in movie.values())
    s = _wall(lambda: graphx.filter_subgraphs(movie, gc.MAP_DICT, gc.PX2ANG), max(3, a.iters // 3))
    print(json.dumps({"what": "e2e", "movie_frames": 100, "atoms": n, "filter_subgraphs_s": round(s, 4)}),
          flush=True)


if __name__ == "__main__":
    main()
