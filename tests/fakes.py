"""Host-side fakes of the device pipeline for the tests of evaluate.py's loop: CUDA events on a counting clock, and
matching, statistics and a packed-call model that record their calls instead of launching anything."""
import torch

import evaluate


class _Event:
    clock = 0.0

    def __init__(self, enable_timing=False):
        self.t = None

    def record(self):
        _Event.clock += 1.0
        self.t = _Event.clock

    def elapsed_time(self, other):
        return (other.t - self.t) * 1000.0           # ms: one second per recorded interval step


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
