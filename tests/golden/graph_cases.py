"""
Seeded inputs of the utils.graphx tests (tests/test_graph*.py, tests/golden/make_golden_graph.py):
jittered graphene honeycombs (C–C 1.42 Å) with Stone–Wales bond rotations (5-7-7-5 rings), an
amorphous patch of random points and a few stray atoms far from the lattice.  Coordinates are in
pixels; PX2ANG converts them to Å.
"""
import numpy as np

PX2ANG = 0.1
MAP_DICT = {0: "C", 1: "Si"}
BOND = 1.42


def honeycomb(nx_: int, ny: int, seed: int, jitter: float = 0.04, n_sw: int = 4,
              patch: float = 6.0, n_stray: int = 5) -> np.ndarray:
    """(N, 3) rows (x, y, class 0) in Å"""
    rng = np.random.default_rng(seed)
    d = BOND
    cell = np.array([[0, 0], [d, 0], [1.5 * d, np.sqrt(3) / 2 * d], [2.5 * d, np.sqrt(3) / 2 * d]])
    ij = np.stack(np.meshgrid(np.arange(nx_), np.arange(ny), indexing="ij"), -1).reshape(-1, 2)
    pos = (ij[:, None, :] * np.array([3 * d, np.sqrt(3) * d]) + cell[None]).reshape(-1, 2)
    span = pos.max(0)
    # Stone–Wales: rotate a horizontal bond (atoms 4c, 4c + 1) by 90° about its midpoint
    inner = [c for c in rng.permutation(len(ij))
             if 2 <= ij[c, 0] < nx_ - 2 and 2 <= ij[c, 1] < ny - 2]
    used = []
    for c in inner:
        if len(used) == n_sw:
            break
        m = pos[4 * c:4 * c + 2].mean(0)
        if any(np.linalg.norm(m - u) < 12 for u in used):
            continue
        used.append(m)
        pos[4 * c] = m + [0, -d / 2]
        pos[4 * c + 1] = m + [0, d / 2]
    pos += rng.normal(0, jitter, pos.shape)
    # amorphous patch: replace a disc by random points at least 1.25 Å apart
    if patch > 0:
        ctr = span * np.array([0.3, 0.7])
        pos = pos[np.linalg.norm(pos - ctr, axis=1) > patch]
        pts = []
        while len(pts) < int(0.33 * np.pi * patch ** 2):
            p = ctr + rng.uniform(-patch, patch, 2)
            if np.linalg.norm(p - ctr) <= patch - 0.4 and \
                    all(np.linalg.norm(p - q) >= 1.25 for q in pts) and \
                    np.min(np.linalg.norm(pos - p, axis=1)) >= 1.25:
                pts.append(p)
        pos = np.concatenate([pos, np.array(pts)])
    stray = span + 8 + rng.uniform(0, 20, (n_stray, 2))
    pos = np.concatenate([pos, stray])
    return np.concatenate([pos, np.zeros((len(pos), 1))], 1)


def single(seed: int = 0) -> np.ndarray:
    """about 2 k C atoms (case 1), in pixels"""
    c = honeycomb(22, 23, seed)
    c[:, :2] /= PX2ANG
    return c


def multi(seed: int = 0) -> np.ndarray:
    """case 1 with about 5 % of the atoms as class 1 (Si)"""
    c = single(seed)
    rng = np.random.default_rng(seed + 100)
    c[rng.random(len(c)) < 0.05, 2] = 1
    return c


def with_z(seed: int = 0) -> np.ndarray:
    """case 1 as (x, y, z, class) with a rippled z"""
    c = single(seed)
    z = 3.0 * np.sin(c[:, 0] * PX2ANG / 9.0) + np.random.default_rng(seed + 200).normal(0, 0.3, len(c))
    return np.concatenate([c[:, :2], z[:, None], c[:, 2:]], 1)


def frames(seed: int = 0) -> dict:
    """three frames for filter_subgraphs; the last one is three separate islands, none of which
    holds half of the atoms"""
    out = {}
    for k in range(2):
        c = honeycomb(10, 10, seed + 10 + k, n_sw=1, patch=3.0, n_stray=4)
        c[:, :2] /= PX2ANG
        out[k] = c
    isl = []
    for k, (w, h) in enumerate([(4, 5), (4, 4), (3, 5)]):
        c = honeycomb(w, h, seed + 20 + k, n_sw=0, patch=0.0, n_stray=0)
        c[:, 0] += 30 * k
        isl.append(c)
    c = np.concatenate(isl)
    c = c[np.random.default_rng(seed + 30).permutation(len(c))]
    c[:, :2] /= PX2ANG
    out[7] = c
    return out


def large(kind: str, seed: int = 0) -> np.ndarray:
    """about 2·10⁴ atoms in pixels: 'lattice' (honeycomb with defects) or 'amorphous' (random
    points at least 1.2 Å apart at close to the densest packing)"""
    if kind == "lattice":
        c = honeycomb(70, 72, seed, n_sw=40, patch=15.0)
    else:
        rng = np.random.default_rng(seed)
        L = 230.0
        p = rng.uniform(0, L, (60000, 2))
        keep = []
        grid = {}
        for i, q in enumerate(p):
            cx, cy = int(q[0] // 1.2), int(q[1] // 1.2)
            ok = True
            for a in (cx - 1, cx, cx + 1):
                for b in (cy - 1, cy, cy + 1):
                    for j in grid.get((a, b), ()):
                        if np.hypot(*(p[j] - q)) < 1.2:
                            ok = False
            if ok:
                grid.setdefault((cx, cy), []).append(i)
                keep.append(i)
            if len(keep) == 20000:
                break
        c = np.concatenate([p[keep], np.zeros((len(keep), 1))], 1)
    c[:, :2] /= PX2ANG
    return c
