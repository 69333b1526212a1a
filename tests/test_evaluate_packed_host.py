"""Host-side logic of evaluate.py --batch_size P > 1: every P pairs go through one `match_many`, one
`PointDSC.forward_packed` and one `eval_stats_packed`, in that order, and the group's device time is split over its pairs."""
import numpy as np
import torch

import evaluate
from test_mixed_batch_host import _Event, _fake_pipeline


class _PackedModel:
    def __init__(self, log):
        self.log = log
        self.calls = []

    def __call__(self, data):
        self.calls.append([data["src_keypts"].shape[1]])
        return {"final_trans": torch.eye(4)[None], "final_labels": torch.ones(1, data["src_keypts"].shape[1])}

    def forward_packed(self, corr_pos, src_keypts, tgt_keypts, offsets, d_offsets=None):
        self.log.append("forward_packed")
        assert d_offsets is not None and d_offsets.tolist() == list(offsets)
        self.calls.append([b - a for a, b in zip(offsets[:-1], offsets[1:])])
        return {"final_trans": torch.eye(4).expand(len(offsets) - 1, 4, 4), "final_labels": torch.ones(offsets[-1])}


def _fake_packed(monkeypatch, log):
    import pointdsc_b200.frontend as fe
    import pointdsc_b200.metrics as me

    def match_many(pairs, use_mutual=False):
        log.append("match_many")
        off = [0]
        for sd, _, _, _ in pairs:
            off.append(off[-1] + int(sd))
        return {"src_keypts": torch.zeros(off[-1], 3), "tgt_keypts": torch.zeros(off[-1], 3), "corr_pos": torch.zeros(off[-1], 6),
                "corr": torch.zeros(off[-1], 2, dtype=torch.int64), "offsets": off, "d_offsets": torch.tensor(off, dtype=torch.int32)}

    def eval_stats_packed(trans, gt, src, tgt, labels, gt_labels, offsets, d_offsets=None, re_thre=15.0, te_thre=30.0):
        log.append("eval_stats_packed")
        assert trans.shape == gt.shape == (len(offsets) - 1, 4, 4) and labels.shape == gt_labels.shape == (offsets[-1],)
        return torch.tensor([[float(b - a)] * 10 for a, b in zip(offsets[:-1], offsets[1:])])

    monkeypatch.setattr(fe, "match_many", match_many)
    monkeypatch.setattr(me, "eval_stats_packed", eval_stats_packed)


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
