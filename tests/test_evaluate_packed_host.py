"""Host-side logic of evaluate.py --batch_size P > 1: every P pairs go through one `match_many`, one
`PointDSC.forward_packed` and one `eval_stats_packed`, in that order, and the group's device time is split over its pairs."""
import numpy as np

import evaluate
from fakes import _Event, _PackedModel, _fake_packed, _fake_pipeline


def test_evaluate_groups_pairs_and_splits_the_model_time(monkeypatch):
    log = []
    _fake_pipeline(monkeypatch)
    _fake_packed(monkeypatch, log)
    cfg = {"inlier_threshold": 0.1, "re_thre": 15.0, "te_thre": 30.0}
    sizes = [30, 40, 50, 60, 70]
    pairs = [(i % 2, (None, n), (None, n), np.eye(4)) for i, n in enumerate(sizes)]
    m = _PackedModel(log)
    out = evaluate.evaluate(m, pairs, cfg, device="cpu", batch_size=2)
    assert m.calls == [[30, 40], [50, 60], [70]]                    # every 2 pairs in one call, the remainder last
    assert log == ["match_many", "forward_packed", "eval_stats_packed"] * 3
    assert out.shape == (5, len(evaluate.COLUMNS))
    assert list(out[:, 0]) == sizes and list(out[:, 11]) == [0, 1, 0, 1, 0]
    assert np.allclose(out[:, 9], [0.5, 0.5, 0.5, 0.5, 1.0])       # the group's device time over its size
    assert (out[:, 10] >= 0).all()
    m1 = _PackedModel(log)
    out1 = evaluate.evaluate(m1, pairs, cfg, device="cpu")
    assert m1.calls == [[n] for n in sizes] and np.allclose(out1[:, 9], 1.0)
    assert np.array_equal(out1[:, :9], out[:, :9])
    assert _Event.clock > 0
