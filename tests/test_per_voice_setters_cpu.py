"""The per-voice setters (set_const_table, set_property_per_voice, set_path_per_voice, set_seq_per_voice) on plan-only runtimes: a
fixed script of per-voice calls, JSON batches and a voice-group cut leaves the render programs, describe() and every voice's
snapshot() exactly as recorded in tests/golden/per_voice_program_words.json; and a failed call of any of the four changes none of
them, also when only a later voice group of the range lacks the node."""
import json
import os
import sys

import numpy as np
import pytest

from elementary_b200 import Runtime, el
from helpers import GOLDEN

sys.path.insert(0, GOLDEN)
import make_per_voice_program_words as script  # noqa: E402

_want = {}


def want(key):
    if not _want:
        with open(os.path.join(GOLDEN, "per_voice_program_words.json")) as f:
            _want.update(json.load(f))
    return _want[key]


@pytest.mark.parametrize("L", script.WIDTHS)
@pytest.mark.parametrize("kind", script.KINDS)
def test_script_matches_recording(kind, L):
    got = json.loads(json.dumps(script.replay(kind, L)))
    recorded = want(f"{kind}/L{L}")
    assert [s["step"] for s in got] == [s["step"] for s in recorded]
    for g, r in zip(got, recorded):
        assert g == r, (kind, L, g["step"])


def two_groups():
    """64 voices in two groups of 32 (tile width 4): every voice has const c, sample s and seq q; the first group also has
    const c1, sample s1 and seq q1."""
    rt = Runtime(script.SR, script.BS, script.VOICES, device=-1, plan_dry_run=1, tile_width=4)
    for name, data in script.RESOURCES.items():
        assert rt.add_shared_resource(name, data)
    base = [el.const(0.5, key="c"), el.sample({"key": "s", "path": "len7"}, el.in_(0)), el.seq({"seq": [1.0, 2.0], "key": "q"}, el.in_(0))]
    extra = [(9001, "const"), (9002, "sample"), (9003, "seq")]
    assert rt.apply_instructions(el.render(*base)) == 0, rt.last_error()
    assert rt.apply_instructions([[0, i, t] for i, t in extra], voices=(0, script.CUT)) == 0, rt.last_error()
    assert len(rt.describe()["groups"]) == 2
    return rt, [n.id() for n in base], [i for i, _ in extra]


def test_failed_calls_change_nothing():
    rt, (c, s, q), (c1, s1, q1) = two_groups()
    # per-voice data already set, so that a failed call would have something to overwrite
    assert rt.set_const_table([c], np.full((1, 64), 2.0, dtype=np.float32)) == 0
    assert rt.set_path_per_voice(s, ["len12"], np.zeros(64)) == 0
    assert rt.set_seq_per_voice(q, [[5.0]], np.zeros(64)) == 0
    before = script.state(rt)
    n = 32   # voices [16, 48): both groups
    table = lambda ids: np.full((len(ids), n), 9.0, dtype=np.float32)  # noqa: E731
    for call, code in [
        (lambda: rt.set_const_table([c, c1], table([c, c1]), voice_begin=16), 2),   # c1 only in the first group
        (lambda: rt.set_const_table([c1], table([c1]), voice_begin=16), 2),
        (lambda: rt.set_const_table([s, c], table([s, c]), voice_begin=16), 5),
        (lambda: rt.set_const_table([c], table([c]), voice_begin=40), -2),         # past the last voice
        (lambda: rt.set_property_per_voice(c1, "value", np.full(n, 9.0), voice_begin=16), 2),
        (lambda: rt.set_property_per_voice(s1, "startOffset", np.full(n, 3.0), voice_begin=16), 2),
        (lambda: rt.set_property_per_voice(s, "startOffset", np.r_[np.full(n - 1, 3.0), -1.0], voice_begin=16), 6),
        (lambda: rt.set_property_per_voice(q, "value", np.full(n, 9.0), voice_begin=16), 5),
        (lambda: rt.set_property_per_voice(c, "value", np.full(n, 9.0), voice_begin=-1), -2),
        (lambda: rt.set_path_per_voice(s1, ["len12"], np.zeros(n), voice_begin=16), 2),
        (lambda: rt.set_path_per_voice(c, ["len12"], np.zeros(n), voice_begin=16), 5),
        (lambda: rt.set_path_per_voice(s, ["len12", "missing"], np.zeros(n), voice_begin=16), 6),
        (lambda: rt.set_seq_per_voice(q1, [[7.0]], np.zeros(n), voice_begin=16), 2),
        (lambda: rt.set_seq_per_voice(s, [[7.0]], np.zeros(n), voice_begin=16), 5),
        (lambda: rt.set_seq_per_voice(q, [[7.0], "text"], np.zeros(n), voice_begin=16), 5),
    ]:
        assert call() == code, rt.last_error()
        assert script.state(rt) == before, code


def test_const_table_missing_in_second_group_changes_nothing():
    """The first group of the range has the const node, the second does not: NodeNotFound, and the first group's rows and its
    snapshot() value are untouched."""
    rt = Runtime(48000.0, 512, 8, device=-1, plan_dry_run=1)
    k = el.const(0.25)
    assert rt.apply_instructions(el.render(el.mul(k, el.in_(0))), voices=(0, 4)) == 0
    assert rt.apply_instructions(el.render(el.cycle(220.0)), voices=(4, 8)) == 0
    assert len(rt.describe()["groups"]) == 2
    before = (rt.describe()["groups"], [rt.snapshot(v) for v in range(8)], rt.program_words(0).tolist())
    assert rt.set_const_table([k.id()], np.full((1, 8), 9.0, dtype=np.float32)) == 2
    assert (rt.describe()["groups"], [rt.snapshot(v) for v in range(8)], rt.program_words(0).tolist()) == before
    assert rt.snapshot(0)[f"0x{k.id() & 0xFFFFFFFF:08x}"]["value"] == 0.25
