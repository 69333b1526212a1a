"""Float64 numpy restatement of FCGF feature extraction (misc/cal_fcgf.py:11-85 with rgb = normal = None, and the ResUNetBN2C
network of misc/fcgf.py:621-867), for tests only.  Sparse tensors are coordinate dictionaries: a level's rows are int coordinates,
and a neighbour is found by looking its coordinate up in the dictionary (a sorted int64 key array and np.searchsorted).

MinkowskiEngine 0.5, which the reference runs the network on, is not a dependency of this project, so its conventions are restated as they are
recalled.  They are numbered as in DESIGN.md (row f8); nothing here can check 4 or 5 against real weights:

  1  Quantisation divides in double: c = floor(x / voxel).  The representative of a voxel is its first point in input order, and
     voxel rows are in first-occurrence order.
  2  A coarser level's coordinates are floor(c / 2s) 2s of the level below (toward -inf for negative c), rows again in
     first-occurrence order over the level below.
  3  For an odd kernel size K the offsets are o in {-r..r}^3, r = (K - 1) / 2, scaled by the input tensor stride for a
     convolution and by the output tensor stride for a transposed convolution.
  4  The kernel index of o is (ox + r) + K (oy + r) + K^2 (oz + r), x fastest.
  5  Convolution: out[q] = sum_o W[o]^T x[q + o s_in].  Transposed convolution: out[q] = sum_o W[o]^T x[q - o s_out] over the
     existing finer coordinates (the strided map transposed).
  6  BatchNorm in eval mode with eps 1e-5.
  7  The output is x / (||x|| + 1e-8).

Coordinates at or beyond 2^20 voxels in magnitude, and non-finite ones, are left out (the device reports them in its status).
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

LIMIT = 1 << 20
BN_EPS = 1e-5

FEAT_WIDTH = {"x0": 32, "t0": 32, "cat0": 96, "d0": 64, "dt0": 64,
              "x1": 64, "t1": 64, "cat1": 128, "d1": 64, "dt1": 64,
              "x2": 128, "t2": 128, "cat2": 256, "d2": 128, "dt2": 128,
              "x3": 256, "t3": 256, "s8": 256}
FEATS = list(FEAT_WIDTH)
FEAT_LEVEL = {f: 3 if f == "s8" else int(f[-1]) for f in FEATS}

# ResUNet2.forward as a list of convolutions: (name, kind, output level, (input buffer, first column) or None,
# (residual buffer, first column) or None, (output buffer, first column), Cout, norm prefix, relu)
STEPS = [
    ("conv1", "c1", 0, None, None, ("x0", 0), 32, "norm1", False),
    ("block1.conv1", "same", 0, ("x0", 0), None, ("t0", 0), 32, "block1.norm1", True),
    ("block1.conv2", "same", 0, ("t0", 0), ("x0", 0), ("cat0", 64), 32, "block1.norm2", True),
    ("conv2", "down", 1, ("cat0", 64), None, ("x1", 0), 64, "norm2", False),
    ("block2.conv1", "same", 1, ("x1", 0), None, ("t1", 0), 64, "block2.norm1", True),
    ("block2.conv2", "same", 1, ("t1", 0), ("x1", 0), ("cat1", 64), 64, "block2.norm2", True),
    ("conv3", "down", 2, ("cat1", 64), None, ("x2", 0), 128, "norm3", False),
    ("block3.conv1", "same", 2, ("x2", 0), None, ("t2", 0), 128, "block3.norm1", True),
    ("block3.conv2", "same", 2, ("t2", 0), ("x2", 0), ("cat2", 128), 128, "block3.norm2", True),
    ("conv4", "down", 3, ("cat2", 128), None, ("x3", 0), 256, "norm4", False),
    ("block4.conv1", "same", 3, ("x3", 0), None, ("t3", 0), 256, "block4.norm1", True),
    ("block4.conv2", "same", 3, ("t3", 0), ("x3", 0), ("s8", 0), 256, "block4.norm2", True),
    ("conv4_tr", "up", 2, ("s8", 0), None, ("d2", 0), 128, "norm4_tr", False),
    ("block4_tr.conv1", "same", 2, ("d2", 0), None, ("dt2", 0), 128, "block4_tr.norm1", True),
    ("block4_tr.conv2", "same", 2, ("dt2", 0), ("d2", 0), ("cat2", 0), 128, "block4_tr.norm2", True),
    ("conv3_tr", "up", 1, ("cat2", 0), None, ("d1", 0), 64, "norm3_tr", False),
    ("block3_tr.conv1", "same", 1, ("d1", 0), None, ("dt1", 0), 64, "block3_tr.norm1", True),
    ("block3_tr.conv2", "same", 1, ("dt1", 0), ("d1", 0), ("cat1", 0), 64, "block3_tr.norm2", True),
    ("conv2_tr", "up", 0, ("cat1", 0), None, ("d0", 0), 64, "norm2_tr", False),
    ("block2_tr.conv1", "same", 0, ("d0", 0), None, ("dt0", 0), 64, "block2_tr.norm1", True),
    ("block2_tr.conv2", "same", 0, ("dt0", 0), ("d0", 0), ("cat0", 0), 64, "block2_tr.norm2", True),
]


def _keys(c: np.ndarray) -> np.ndarray:
    c = np.asarray(c, np.int64) + LIMIT
    return (c[:, 0] << 42) | (c[:, 1] << 21) | c[:, 2]


def first_occurrence(c: np.ndarray) -> np.ndarray:
    """Indices of the first row of every distinct coordinate of c [n,3], in order of first occurrence."""
    if len(c) == 0:
        return np.zeros(0, np.int64)
    _, first = np.unique(_keys(c), return_index=True)
    return np.sort(first)


def quantize(xyz: np.ndarray, voxel: float) -> Tuple[np.ndarray, np.ndarray, bool]:
    """(coords [m,3] int64, representative indices [m], any point left out): conventions 1 and the +-2^20 bound."""
    f = np.floor(np.asarray(xyz, np.float64) / float(voxel))
    ok = np.all(np.isfinite(f) & (f >= -LIMIT) & (f < LIMIT), axis=1)
    idx = np.nonzero(ok)[0]
    c = f[idx].astype(np.int64)
    first = first_occurrence(c)
    return c[first], idx[first], bool((~ok).any())


def pyramid(coords0: np.ndarray, levels: int = 4) -> List[np.ndarray]:
    """Coordinates of tensor strides 1, 2, 4, 8 (convention 2)."""
    out = [np.asarray(coords0, np.int64)]
    for l in range(1, levels):
        c = np.floor_divide(out[-1], 2 ** l) * 2 ** l
        out.append(c[first_occurrence(c)])
    return out


def offsets(K: int) -> np.ndarray:
    """[K^3, 3] offsets in kernel-index order (conventions 3 and 4: x fastest)."""
    r = (K - 1) // 2
    o = np.arange(K ** 3)
    return np.stack([o % K - r, (o // K) % K - r, o // (K * K) - r], axis=1)


def kernel_map(out_coords: np.ndarray, table: np.ndarray, K: int, mult: int) -> np.ndarray:
    """[m, K^3] int64: the row of `table` at out_coords[q] + o * mult, or -1."""
    keys = _keys(table)
    order = np.argsort(keys)
    sk = keys[order]
    res = np.full((len(out_coords), K ** 3), -1, np.int64)
    for o, d in enumerate(offsets(K)):
        q = np.asarray(out_coords, np.int64) + d * mult
        ok = np.all((q >= -LIMIT) & (q < LIMIT), axis=1)
        k = _keys(np.where(ok[:, None], q, 0))
        pos = np.minimum(np.searchsorted(sk, k), len(sk) - 1)
        hit = ok & (sk[pos] == k) if len(sk) else np.zeros(len(q), bool)
        res[hit, o] = order[pos[hit]]
    return res


def maps(levels: Sequence[np.ndarray], k1: int) -> Dict[str, np.ndarray]:
    """Every neighbour table of the network: c1, same<l>, down<l> (l = 1..3), up<l> (l = 0..2)."""
    m = {"c1": kernel_map(levels[0], levels[0], k1, 1)}
    for l in range(4):
        m[f"same{l}"] = kernel_map(levels[l], levels[l], 3, 2 ** l)
    for l in range(1, 4):
        m[f"down{l}"] = kernel_map(levels[l], levels[l - 1], 3, 2 ** (l - 1))
    for l in range(3):
        m[f"up{l}"] = kernel_map(levels[l], levels[l + 1], 3, -(2 ** l))
    return m


def step_map(step, mp: Dict[str, np.ndarray]) -> np.ndarray:
    kind, level = step[1], step[2]
    return mp["c1"] if kind == "c1" else mp[f"{kind}{level}"]


def sparse_conv(x: np.ndarray, nmap: np.ndarray, W: np.ndarray) -> np.ndarray:
    """sum over offsets o of W[o]^T x[map[:, o]] (absent neighbours contribute nothing), float64."""
    W = np.asarray(W, np.float64)
    out = np.zeros((nmap.shape[0], W.shape[2]))
    for o in range(nmap.shape[1]):
        rows = np.nonzero(nmap[:, o] >= 0)[0]
        if len(rows):
            out[rows] += x[nmap[rows, o]] @ W[o]
    return out


def batch_norm(x: np.ndarray, sd: Dict[str, np.ndarray], prefix: str) -> np.ndarray:
    g, b = (np.asarray(sd[f"{prefix}.bn.{k}"], np.float64) for k in ("weight", "bias"))
    mu, var = (np.asarray(sd[f"{prefix}.bn.{k}"], np.float64) for k in ("running_mean", "running_var"))
    return (x - mu) / np.sqrt(var + BN_EPS) * g + b


def apply_step(step, sd, nmap: np.ndarray, x_in: np.ndarray, residual) -> np.ndarray:
    """One convolution with its BN, residual and ReLU (x_in: the input columns, or None for conv1's constant 1)."""
    name = step[0]
    W = np.asarray(sd[f"{name}.kernel"], np.float64)
    if x_in is None:                                   # conv1 reads level 0 itself: one 1.0 per row
        x_in = np.ones((nmap.shape[0], 1))
    y = batch_norm(sparse_conv(x_in, nmap, W), sd, step[7])
    if residual is not None:
        y = y + residual
    return np.maximum(y, 0.0) if step[8] else y


def head(cat0: np.ndarray, sd) -> np.ndarray:
    """conv1_tr, ReLU, final (+ bias), x / (||x|| + 1e-8)."""
    w_tr = np.asarray(sd["conv1_tr.kernel"], np.float64).reshape(96, 64)
    w_f = np.asarray(sd["final.kernel"], np.float64).reshape(64, 32)
    f = np.maximum(cat0 @ w_tr, 0.0) @ w_f + np.asarray(sd["final.bias"], np.float64).reshape(32)
    return f / (np.linalg.norm(f, axis=1, keepdims=True) + 1e-8)


def forward(sd, levels: Sequence[np.ndarray], k1: int, mp=None) -> Tuple[np.ndarray, Dict[str, np.ndarray]]:
    """(descriptors [m0,32], every feature buffer) of ResUNetBN2C over the coordinate levels, float64."""
    mp = maps(levels, k1) if mp is None else mp
    buf = {f: np.zeros((len(levels[FEAT_LEVEL[f]]), w)) for f, w in FEAT_WIDTH.items()}
    for step in STEPS:
        x = None if step[3] is None else buf[step[3][0]][:, step[3][1]:]
        res = None if step[4] is None else buf[step[4][0]][:, step[4][1]:step[4][1] + step[6]]
        y = apply_step(step, sd, step_map(step, mp), x, res)
        buf[step[5][0]][:, step[5][1]:step[5][1] + step[6]] = y
    return head(buf["cat0"], sd), buf


def extract_features(sd, xyz: np.ndarray, voxel: float, k1: int):
    """(key points xyz[inds], descriptors [m,32] float64) as misc/cal_fcgf.py's extract_features returns them."""
    c0, inds, _ = quantize(xyz, voxel)
    desc, _ = forward(sd, pyramid(c0), k1)
    return np.asarray(xyz)[inds], desc
