"""Cost of utils.imgen's lattice masks and of extract_patches_ on the GPU (csrc/imgen.cu, the patch
gather of csrc/frontend.cu).

  kernel  CUDA-event ms of the owner, fill and gather passes, averaged over --iters launches after
          a warm-up, with the bytes each pass moves (model below) and GB/s against the H100 SXM's
          3.35 TB/s
  e2e     wall time of the public call, ending in a device synchronise, median of --iters calls:
          numpy in / numpy out and CUDA in / CUDA out; and the host restatement's per-atom slice
          loop (oracle/imgen_ref.py), which is how the reference spends its time, in the same run
Bytes model: owner = the atom rows (36 B each) + 8 B (an atomic's read and write) per slice pixel;
fill = the owner planes (4 B per pixel and class) + the output; gather = the patches read + written.
Template and atom-row reads by the fill pass hit in cache and are left out.  Overlapping patches
reread image rows that L2 serves, so the gather's model rate can exceed the HBM bandwidth.
Workloads: a 1024² frame of 15 876 atoms in 2 classes; 100 frames of 512² with 3 844 atoms each in
3 classes; extract_patches_ of 500 patches of 256² from a 2048² float64 image and a
(2048, 2048, 3) float64 mask.  Prints the card's name and power limit, then one JSON line per
measurement.

    python tools/bench_imgen.py [--iters 10]
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

import imgen_cases as ic  # noqa: E402
from atomai_b200 import _C, ops, utils  # noqa: E402
from oracle import imgen_ref  # noqa: E402

PEAK = 3.35e12


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


def _capture(name, call):
    """the arguments of every ops.<name> call `call` makes, in order"""
    seen, orig = [], getattr(ops, name)

    def spy(*a):
        seen.append(a)
        return orig(*a)
    setattr(ops, name, spy)
    try:
        call()
    finally:
        setattr(ops, name, orig)
    return seen


def _emit(**kw):
    print(json.dumps(kw), flush=True)


def masks(tag, imgs, coords, iters):
    lib, st = _C.lib(), _C.stream_ptr
    call = lambda: utils.create_multiclass_lattice_mask(imgs, {k: v.copy() for k, v in coords.items()})
    atoms, frames, max_pix, owner, tpl, out, bg = _capture("imgen_masks", call)[0]
    nr, nc = atoms[:, 4].long(), atoms[:, 5].long()
    K, F = atoms.shape[0], frames.shape[0]

    def owner_pass():
        owner.zero_()
        _C.check(lib.atomai_b200_imgen_owner(_C.ptr(atoms), K, _C.ptr(frames), _C.ptr(owner), st()))

    def fill_pass():
        _C.check(lib.atomai_b200_imgen_fill(_C.ptr(atoms), _C.ptr(frames), F, max_pix,
                                            _C.ptr(owner), _C.ptr(tpl), 8, int(bg), _C.ptr(out),
                                            st()))
    zero_ms = _events(owner.zero_, iters)
    for name, fn, nbytes in (
            ("owner", owner_pass, K * 36 + 8 * int((nr * nc).sum())),
            ("fill", fill_pass, owner.numel() * 4 + out.numel() * 8)):
        ms = _events(fn, iters) - (zero_ms if name == "owner" else 0.0)
        _emit(workload=tag, measure=f"{name}_kernel", ms=round(ms, 4), bytes=nbytes,
              gbps=round(nbytes / ms / 1e6, 1), share_of_peak=round(nbytes / ms / 1e-3 / PEAK, 3))
    _emit(workload=tag, measure="owner_memset", ms=round(zero_ms, 4), bytes=owner.numel() * 4)
    dev = torch.from_numpy(imgs).cuda()
    cuda_call = lambda: utils.create_multiclass_lattice_mask(
        dev, {k: v.copy() for k, v in coords.items()})
    _emit(workload=tag, measure="wall_numpy", ms=round(_wall(call, iters) * 1e3, 2))
    _emit(workload=tag, measure="wall_cuda", ms=round(_wall(cuda_call, iters) * 1e3, 2))
    t0 = time.perf_counter()
    ref = [imgen_ref.multiclass_mask(im.shape, coords[i], utils.create_atom_mask_pair)
           for i, im in enumerate(imgs)]
    host_s = time.perf_counter() - t0
    same = np.stack(ref).tobytes() == np.asarray(call()).tobytes()
    _emit(workload=tag, measure="oracle_host_loop", ms=round(host_s * 1e3, 1), equal=same)


def patches(iters):
    tag = "patches_500x256_from_2048"
    rng = np.random.default_rng(0)
    im = rng.random((2048, 2048))
    mask = rng.random((2048, 2048, 3))
    call = lambda: utils.extract_patches_(im, mask, 256, 500, random_state=0)
    # extract_patches_ gathers the image patches first, then the mask patches
    for what, (img, offs, ph, pw, out) in zip(("image", "mask"), _capture("gather_patches", call)):
        nbytes = 2 * out.numel() * out.element_size()
        ms = _events(lambda: ops.gather_patches(img, offs, ph, pw, out), iters)
        _emit(workload=tag, measure=f"gather_kernel_{what}", ms=round(ms, 4), bytes=nbytes,
              gbps=round(nbytes / ms / 1e6, 1),
              share_of_peak=round(nbytes / ms / 1e-3 / PEAK, 3))
    di, dm = torch.from_numpy(im).cuda(), torch.from_numpy(mask).cuda()
    _emit(workload=tag, measure="wall_numpy", ms=round(_wall(call, iters) * 1e3, 2))
    _emit(workload=tag, measure="wall_cuda", ms=round(_wall(
        lambda: utils.extract_patches_(di, dm, 256, 500, random_state=0), iters) * 1e3, 2))
    t0 = time.perf_counter()
    rs = np.random.RandomState(0)
    i, j = rs.randint(2048 - 255, size=500), rs.randint(2048 - 255, size=500)
    ref_im = np.stack([im[a:a + 256, b:b + 256] for a, b in zip(i, j)])
    rs = np.random.RandomState(0)
    i, j = rs.randint(2048 - 255, size=500), rs.randint(2048 - 255, size=500)
    ref_lb = np.stack([mask[a:a + 256, b:b + 256] for a, b in zip(i, j)])
    host_s = time.perf_counter() - t0
    got = call()
    same = got[0].tobytes() == ref_im.tobytes() and got[1].tobytes() == ref_lb.tobytes()
    _emit(workload=tag, measure="host_slice_loop", ms=round(host_s * 1e3, 1), equal=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"card: {q}", flush=True)
    one = {0: ic.with_classes(ic.square(126, 8.0, 1, jitter=0.4, origin=6.0), [0, 1], 1)}
    masks("frame_1024_16k_2cls", np.zeros((1, 1024, 1024), np.float32), one, a.iters)
    stack = {i: ic.with_classes(ic.square(62, 8.0, 10 + i, jitter=0.4, origin=6.0), [1, 2, 3], i)
             for i in range(100)}
    masks("stack_100x512_4k_3cls", np.zeros((100, 512, 512), np.float32), stack, a.iters)
    patches(a.iters)


if __name__ == "__main__":
    main()
