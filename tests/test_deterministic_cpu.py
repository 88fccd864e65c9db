"""Deterministic mode on the CPU test double: every engine and player call sets the library's mode from torch's switch
through `sync_deterministic`; the Dreamer-V3 step-graph key holds the mode; and with the switch off the op sequence an
engine issues is the one it issued before the mode existed (the same trace as with the mode's setter absent)."""
import pytest
import torch

from oracle.ops_emul import EmulOps


@pytest.fixture
def switch():
    """sets torch's switch for one test and restores it"""
    was = torch.are_deterministic_algorithms_enabled()

    def set_(on):
        torch.use_deterministic_algorithms(on)

    yield set_
    torch.use_deterministic_algorithms(was)


class RecordingOps(EmulOps):
    """the test double with the library's setter, which records each mode it is given"""

    def __init__(self):
        super().__init__()
        self.modes = []

    def set_deterministic(self, on):
        self.modes.append(bool(on))


def test_sync_follows_torch_switch(switch):
    from sheeprl_b200.lib import sync_deterministic

    ops = RecordingOps()
    switch(True)
    assert sync_deterministic(ops) is True
    switch(False)
    assert sync_deterministic(ops) is False
    assert ops.modes == [True, False]
    assert sync_deterministic(EmulOps()) is False          # a backend without the setter is left alone


def _scenarios():
    from tests.op_trace import _tool, dv3_scenarios

    return list(_tool().scenarios()) + list(dv3_scenarios())


SCENARIOS = dict(_scenarios())


@pytest.mark.parametrize("title", sorted(SCENARIOS))
def test_every_entry_point_sets_the_mode(switch, monkeypatch, title):
    """every engine train(), public train() wrapper and player of the fixture configurations sets the library mode from
    torch's switch (the setter on the test double records it)"""
    seen = []
    monkeypatch.setattr(EmulOps, "set_deterministic", lambda self, on: seen.append(bool(on)), raising=False)
    switch(True)                    # off is the default every other CPU test runs with
    try:
        SCENARIOS[title]()
    except AssertionError:
        pass                        # fixture tolerances are not what is checked here
    assert seen and set(seen) == {True}, (title, seen[:3])


def test_dv3_graph_key_holds_the_mode(switch):
    from sheeprl_b200.configs import make_dv3_cfg
    from sheeprl_b200.engine import DV3Engine

    cfg = make_dv3_cfg("S", per_rank_batch_size=2, per_rank_sequence_length=4, horizon=3, dense_units=16, mlp_layers=1,
                       cnn_channels_multiplier=4, recurrent_state_size=16, hidden_size=16, stochastic_size=4,
                       discrete_size=4, bins=15)
    eng = DV3Engine(cfg, (3,), in_channels=3, device="cpu", ops=RecordingOps())
    switch(False)
    off = eng.graph_key()
    switch(True)
    on = eng.graph_key()
    assert off != on and off[:-1] == on[:-1]


def test_switch_off_issues_the_ops_of_the_parent_commit(switch):
    """tests/golden/op_trace_default.json: the op-sequence digests of every scenario of tests/op_trace.py, recorded at
    the commit before the deterministic mode existed; with the switch off every engine and player issues that sequence"""
    import json
    import os

    from tests.op_trace import digests

    switch(False)
    with open(os.path.join(os.path.dirname(__file__), "golden", "op_trace_default.json")) as f:
        want = json.load(f)
    got = digests()
    assert sorted(got) == sorted(want)
    assert [k for k in want if got[k] != want[k]] == []
