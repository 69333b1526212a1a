"""Host-side logic of mixed-size calls: PointDSC.forward_many's argument checks (raised before any engine call) and the
grouping of evaluate.py --batch_size."""
import numpy as np
import pytest
import torch

import evaluate
from fakes import _fake_pipeline
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


class _Model:
    def __init__(self):
        self.calls = []

    def __call__(self, data):
        self.calls.append([data["src_keypts"].shape[1]])
        return {"final_trans": torch.eye(4)[None], "final_labels": torch.ones(1, data["src_keypts"].shape[1])}

    def forward_many(self, batches):
        self.calls.append([b["src_keypts"].shape[1] for b in batches])
        return [{"final_trans": torch.eye(4)[None], "final_labels": torch.ones(1, b["src_keypts"].shape[1])} for b in batches]


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
