"""The float64 restatement of the spectral-matching baseline (oracle/sm_oracle.py), on the CPU.

Against the reference's own `SM` (baseline_scripts/baseline_3DMatch.py:19-53), run in torch fp32 where a checkout of the reference
is named by POINTDSC_REFERENCE (skipped otherwise).  That module imports open3d and the data loaders at its top, so only the `SM`
function is taken from it: its source is parsed with `ast` and that one definition is executed, with `rigid_transform_3d` taken
the same way from models/common.py.  Then the edge families: S = 0 (N < 10), all rows outliers, duplicate rows, all inliers.
"""
import ast
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import sm_oracle as O
from pointdsc_b200.synth import make_pair

REF = os.environ.get("POINTDSC_REFERENCE")


def _function(path, name, namespace):
    tree = ast.parse(open(path).read(), filename=path)
    node = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name)
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), namespace)
    return namespace[name]


@pytest.fixture(scope="module")
def reference_sm():
    if not REF or not os.path.exists(os.path.join(REF, "baseline_scripts", "baseline_3DMatch.py")):
        pytest.skip("POINTDSC_REFERENCE does not name a checkout of the reference")
    sys.path.insert(0, REF)
    try:
        from utils.SE3 import integrate_trans
    finally:
        sys.path.remove(REF)
    ns = {"torch": torch, "integrate_trans": integrate_trans}
    rigid = _function(os.path.join(REF, "models", "common.py"), "rigid_transform_3d", ns)
    ns["rigid_transform_3d"] = rigid
    return _function(os.path.join(REF, "baseline_scripts", "baseline_3DMatch.py"), "SM", ns)


@pytest.mark.parametrize("preset,n,seed,ratio", [("3dmatch", 200, 0, 0.3), ("3dmatch", 1000, 1, 0.1), ("3dmatch", 517, 2, 0.6),
                                                 ("kitti", 400, 3, 0.3), ("kitti", 1000, 4, 0.5)])
def test_oracle_agrees_with_reference_sm(reference_sm, preset, n, seed, ratio):
    thr = 0.10 if preset == "3dmatch" else 0.6
    p = make_pair(seed, n, preset, ratio)
    trans, labels = reference_sm(p["corr_pos"][None], p["src_keypts"][None], p["tgt_keypts"][None],
                                 SimpleNamespace(inlier_threshold=thr))
    o = O.sm(p["corr_pos"], p["src_keypts"], p["tgt_keypts"], thr)
    # the reference's fp32 v is within a few hundred fp32 roundings of float64 on these sets; its labels agree wherever the
    # float64 selection gap is wider than that, and its T is that of (nearly) the same weights
    assert o["S"] == int(n * 0.1)
    if o["gap"] > 1e-4:
        assert torch.equal(labels[0].double(), o["labels"]), (o["gap"], int((labels[0].double() != o["labels"]).sum()))
    else:
        assert int((labels[0].double() != o["labels"]).sum()) <= 4
    assert np.abs(trans[0].double().numpy() - o["trans"].numpy()).max() < 1e-3


def test_s_zero_is_identity():
    for n in range(2, 10):
        p = make_pair(n, n, "3dmatch", 0.5)
        o = O.sm(p["corr_pos"], p["src_keypts"], p["tgt_keypts"], 0.10)
        assert o["S"] == 0 and o["labels"].sum() == 0 and o["gap"] == math.inf
        assert torch.equal(o["H"], torch.zeros(3, 3, dtype=torch.float64))
        assert torch.equal(o["trans"], torch.eye(4, dtype=torch.float64))


def test_all_outliers_v_zero_after_one_step():
    """Rows whose pairwise length differences all exceed the threshold: M = 0, so v = 0 after the first step and T = I."""
    n = 40
    i = torch.arange(n, dtype=torch.float32)
    src = torch.stack([i, torch.zeros(n), torch.zeros(n)], 1)            # spacing 1 on a line
    tgt = torch.stack([3.0 * i, torch.zeros(n), torch.zeros(n)], 1)      # spacing 3: |m| >= 2 > tau for every pair
    corr = torch.cat([src, tgt], 1)
    corr = corr - corr.mean(0)
    o = O.sm(corr, src, tgt, 0.10)
    assert torch.equal(o["M"], torch.zeros(n, n, dtype=torch.float64))
    assert torch.equal(o["iterates"][1], torch.zeros(n, dtype=torch.float64)) and torch.equal(o["v"], o["iterates"][1])
    assert o["S"] == 4 and o["labels"][:4].sum() == 4                     # ties: the lowest rows
    assert torch.equal(o["trans"], torch.eye(4, dtype=torch.float64))


def test_duplicate_rows():
    """Repeated rows: a row and its copy have the same v up to the order of the float64 sums, and the selection is the stable
    descending order of v (exact ties, lowest row first, are covered by the all-outlier set)."""
    p = make_pair(7, 50, "3dmatch", 0.4)
    c, s, t = p["corr_pos"].clone(), p["src_keypts"].clone(), p["tgt_keypts"].clone()
    c[25:], s[25:], t[25:] = c[:25], s[:25], t[:25]
    o = O.sm(c, s, t, 0.10)
    v = o["v"]
    assert torch.allclose(v[:25], v[25:], rtol=1e-12, atol=1e-15)
    assert (v[o["labels"] == 1].min() >= v[o["labels"] == 0].max()) and o["labels"].sum() == 5


def test_all_inliers_recover_the_motion():
    p = make_pair(11, 300, "3dmatch", 1.0)
    o = O.sm(p["corr_pos"], p["src_keypts"], p["tgt_keypts"], 0.10)
    assert o["S"] == 30 and o["labels"].sum() == 30 and (o["v"] > 0).all()
    gt = p["gt_trans"].double()
    assert (o["trans"][:3, :3] - gt[:3, :3]).abs().max() < 0.05 and (o["trans"][:3, 3] - gt[:3, 3]).abs().max() < 0.05
