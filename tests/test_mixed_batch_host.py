"""Host-side logic of mixed-size calls: PointDSC.forward_many's argument checks (raised before any engine call) and the
grouping of evaluate.py --batch_size."""
import numpy as np
import pytest
import torch

import evaluate
from pointdsc_b200 import PointDSC


def _batch(bs, n, testing=True):
    d = {"corr_pos": torch.zeros(bs, n, 6), "src_keypts": torch.zeros(bs, n, 3), "tgt_keypts": torch.zeros(bs, n, 3)}
    if testing:
        d["testing"] = True
    return d


def test_forward_many_rejects_bad_batches_before_the_engine():
    m = PointDSC()
    with pytest.raises(ValueError, match="testing"):
        m.forward_many([_batch(1, 20, testing=False)])
    bad = _batch(1, 20)
    bad["src_keypts"] = torch.zeros(1, 19, 3)
    with pytest.raises(ValueError, match="expected corr_pos"):
        m.forward_many([bad, _batch(1, 30)])
    bad = _batch(1, 20)
    bad["corr_pos"] = torch.zeros(1, 20, 5)
    with pytest.raises(ValueError, match="expected corr_pos"):
        m.forward_many([bad])
    with pytest.raises(ValueError, match="device tensors"):      # host tensors
        m.forward_many([_batch(2, 20)])
    assert m._engine is None
    assert m.forward_many([]) == []


class _Event:
    clock = 0.0

    def __init__(self, enable_timing=False):
        self.t = None

    def record(self):
        _Event.clock += 1.0
        self.t = _Event.clock

    def elapsed_time(self, other):
        return (other.t - self.t) * 1000.0           # ms: one second per recorded interval step


class _Model:
    def __init__(self):
        self.calls = []

    def __call__(self, data):
        self.calls.append([data["src_keypts"].shape[1]])
        return {"final_trans": torch.eye(4)[None], "final_labels": torch.ones(1, data["src_keypts"].shape[1])}

    def forward_many(self, batches):
        self.calls.append([b["src_keypts"].shape[1] for b in batches])
        return [{"final_trans": torch.eye(4)[None], "final_labels": torch.ones(1, b["src_keypts"].shape[1])} for b in batches]


def _fake_pipeline(monkeypatch):
    import pointdsc_b200.frontend as fe
    import pointdsc_b200.metrics as me

    def match(src_desc, tgt_desc, src_xyz, tgt_xyz, use_mutual=False):
        n = int(src_desc)
        return {"src_keypts": torch.zeros(1, n, 3), "tgt_keypts": torch.zeros(1, n, 3), "corr_pos": torch.zeros(1, n, 6)}

    def eval_stats(trans, gt, src, tgt, labels, gt_labels, re_thre, te_thre):
        return torch.full((1, 10), float(src.shape[1]))

    monkeypatch.setattr(fe, "match", match)
    monkeypatch.setattr(me, "eval_stats", eval_stats)
    monkeypatch.setattr(evaluate, "gt_labels", lambda data, gt, thr: torch.ones(1, data["src_keypts"].shape[1]))
    monkeypatch.setattr(torch.cuda, "Event", _Event)


def test_evaluate_groups_pairs_and_splits_the_model_time(monkeypatch):
    _fake_pipeline(monkeypatch)
    cfg = {"inlier_threshold": 0.1, "re_thre": 15.0, "te_thre": 30.0}
    sizes = [30, 40, 50, 60, 70]
    pairs = [(i % 2, (None, n), (None, n), np.eye(4)) for i, n in enumerate(sizes)]
    m = _Model()
    out = evaluate.evaluate(m, pairs, cfg, device="cpu", batch_size=2)
    assert m.calls == [[30, 40], [50, 60], [70]]                    # every 2 pairs in one call, the remainder last
    assert out.shape == (5, len(evaluate.COLUMNS))
    assert list(out[:, 0]) == sizes and list(out[:, 11]) == [0, 1, 0, 1, 0]
    assert np.allclose(out[:, 9], [0.5, 0.5, 0.5, 0.5, 1.0])       # the group's device time over its size
    m1 = _Model()
    out1 = evaluate.evaluate(m1, pairs, cfg, device="cpu")
    assert m1.calls == [[n] for n in sizes] and np.allclose(out1[:, 9], 1.0)
    assert np.array_equal(out1[:, :9], out[:, :9])
