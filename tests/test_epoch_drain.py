"""The synchronous forms of EpochProcessor (process_epoch_dev, process_epoch_host, get_head) share slot 0 and the vote accumulator
with the pipeline, so they refuse to run while submitted epochs are in flight: AssertionError before anything is enqueued.  After
drain() they run as usual.  CPU only: a stand-in engine records its calls, torch's stream and event calls are stubbed."""
import numpy as np
import pytest
import torch

N_AGG, N_SIG, N_BLK, DEPTH = 4, 8, 10, 3


class _Stream:
    def wait_event(self, ev):
        pass

    def synchronize(self):
        pass


class _Event:
    def record(self, stream=None):
        pass

    def synchronize(self):
        pass


class _Engine:
    """Stand-in for engine.Engine: every verdict 1, head = the justified index; every call recorded by name."""
    device = 0

    def __init__(self):
        self.calls = []

    def epoch_set_pairing_form(self, team):
        self.calls.append("epoch_set_pairing_form")

    def epoch_start_dev(self, slot, d_sigs, d_members, d_off, d_bits, d_msgs, d_agg_status):
        self.calls.append("epoch_start_dev")

    def epoch_tail_dev(self, slot, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        d_ok.fill_(1)
        self.calls.append("epoch_tail_dev")

    def epoch_wait_dev(self, slot):
        self.calls.append("epoch_wait_dev")

    def epoch_dev(self, d_sigs, d_members, d_off, d_bits, d_msgs, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        d_ok.fill_(1)
        self.calls.append("epoch_dev")

    def vote_weights_dev(self, d_votes):
        self.calls.append("vote_weights_dev")

    def head_from_votes_dev(self, d_votes, d_head, justified_idx=0, boost_idx=-1, boost_score=0):
        d_head[0] = justified_idx
        self.calls.append("head_from_votes_dev")


def test_synchronous_calls_need_a_drained_pipeline(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    from pos_evolution_b200.epoch import EpochProcessor
    eng = _Engine()
    ep = EpochProcessor(eng, N_AGG, N_SIG, 1, N_BLK, device=torch.device("cpu"), depth=DEPTH)
    ep.set_committees(np.arange(N_SIG, dtype=np.uint32), (np.arange(N_AGG + 1) * 2).astype(np.uint32))
    args = (torch.zeros((N_SIG, 96), dtype=torch.uint8), torch.zeros((N_AGG, 1), dtype=torch.uint8), torch.zeros((N_AGG, 32), dtype=torch.uint8),
            torch.zeros(N_AGG, dtype=torch.int64), torch.zeros(N_AGG, dtype=torch.int32))
    assert ep.submit_dev(*args) is None and ep.submit_dev(*args) is None
    calls, k = list(eng.calls), ep.k
    for call in (lambda: ep.process_epoch_dev(*args, 5), lambda: ep.process_epoch_host(*args, 5), lambda: ep.get_head(5)):
        with pytest.raises(AssertionError):
            call()
        assert eng.calls == calls and ep.k == k             # nothing enqueued
    tickets = ep.drain()
    assert len(tickets) == 2 and all(t.wait()[0].tolist() == [1] * N_AGG for t in tickets)
    ok, head = ep.process_epoch_dev(*args, 5)
    assert ok.tolist() == [1] * N_AGG and int(head[0]) == 5
    ok, head = ep.process_epoch_host(*args, 6)
    assert ok.tolist() == [1] * N_AGG and head == 6
    assert ep.get_head(7) == 7
    assert eng.calls[len(calls):] == ["epoch_dev", "vote_weights_dev", "head_from_votes_dev"] * 2 + ["vote_weights_dev", "head_from_votes_dev"]
