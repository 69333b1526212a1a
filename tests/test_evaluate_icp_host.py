"""Host-side logic of evaluate.py --use_icp: the transform is refined after the forward and before the statistics, inside the
model-time events, once per pair (bs = 1) or once per packed group; without the flag ICP never runs."""
import numpy as np
import pytest
import torch

import evaluate
from test_evaluate_packed_host import _PackedModel, _fake_packed
from test_mixed_batch_host import _fake_pipeline


def _fake_icp(monkeypatch, log):
    import pointdsc_b200.icp as icp
    import pointdsc_b200.metrics as me

    def icp_refine(src, tgt, trans, max_correspondence_distance=0.10):
        log.append("icp_refine")
        assert max_correspondence_distance == 0.10 and trans.shape == (1, 4, 4)
        return trans * 2.0

    def icp_refine_packed(src, tgt, trans, offsets, d_offsets=None, max_correspondence_distance=0.10, max_iteration=30, info=False):
        log.append("icp_refine_packed")
        assert d_offsets is not None and trans.shape == (len(offsets) - 1, 4, 4) and src.shape == (offsets[-1], 3)
        return trans * 2.0

    def eval_stats(trans, gt, src, tgt, labels, gt_labels, re_thre, te_thre):
        log.append("eval_stats")
        return torch.full((1, 10), float(trans[0, 0, 0]))

    packed_stats = me.eval_stats_packed

    def eval_stats_packed(trans, *args, **kw):
        out = packed_stats(trans, *args, **kw)
        out[:, 1] = trans[:, 0, 0]
        return out

    monkeypatch.setattr(icp, "icp_refine", icp_refine)
    monkeypatch.setattr(icp, "icp_refine_packed", icp_refine_packed)
    monkeypatch.setattr(me, "eval_stats", eval_stats)
    monkeypatch.setattr(me, "eval_stats_packed", eval_stats_packed)


class _LoggedModel(_PackedModel):
    def __call__(self, data):
        self.log.append("forward")
        return super().__call__(data)


@pytest.mark.parametrize("use_icp", [False, True])
def test_icp_runs_between_forward_and_statistics(monkeypatch, use_icp):
    log = []
    _fake_pipeline(monkeypatch)
    _fake_packed(monkeypatch, log)
    _fake_icp(monkeypatch, log)
    events = []
    record = evaluate.torch.cuda.Event.record

    def logged_record(self):
        events.append(len(log))
        record(self)
    monkeypatch.setattr(evaluate.torch.cuda.Event, "record", logged_record)
    cfg = {"inlier_threshold": 0.1, "re_thre": 15.0, "te_thre": 30.0}
    sizes = [30, 40, 50]
    pairs = [(0, (None, n), (None, n), np.eye(4)) for n in sizes]

    log.clear()
    out1 = evaluate.evaluate(_LoggedModel(log), pairs, cfg, device="cpu", use_icp=use_icp)
    step = ["forward", "icp_refine", "eval_stats"] if use_icp else ["forward", "eval_stats"]
    assert log == step * 3
    # the events of pair p enclose its forward and its ICP, not its statistics
    for p in range(3):
        a, b = events[2 * p], events[2 * p + 1]
        assert log[a:b] == step[:-1]
    assert list(out1[:, 0]) == [2.0 if use_icp else 1.0] * 3

    log.clear()
    events.clear()
    out4 = evaluate.evaluate(_PackedModel(log), pairs, cfg, device="cpu", batch_size=2, use_icp=use_icp)
    step = ["match_many", "forward_packed"] + (["icp_refine_packed"] if use_icp else []) + ["eval_stats_packed"]
    assert log == step * 2
    for g in range(2):
        a, b = events[2 * g], events[2 * g + 1]
        assert log[a:b] == step[1:-1]
    assert list(out4[:, 1]) == [2.0 if use_icp else 1.0] * 3


def test_use_icp_flag():
    assert evaluate.parse_args([]).use_icp is False
    assert evaluate.parse_args(["--use_icp"]).use_icp is True
