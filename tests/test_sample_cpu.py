"""The `sample` node without a GPU: its props' return codes, the render program it compiles to, the per-voice entry points'
argument checks, and SampleModel (tests/sample_common.py, what the GPU tests compare with) against the compiled reference in every
scenario the GPU tests render.  Where oracle/_ref is absent the reference's results come from tests/golden/reference_sample.npz."""
import json
import os

import numpy as np
import pytest

from elementary_b200 import Runtime, el
from helpers import GOLDEN
from oracle import oracle as orc
import sample_common
from sample_common import BS, SR

OP_END, OP_SEG, OP_CUSTOM, OP_SAMPLE = 0, 1, 42, 43    # program.h: OP_SAMPLE comes after every opcode that existed before it

PROP_CASES = [
    ("path", 3.0), ("path", "missing"), ("path", "len7"), ("path", "len7"), ("path", True),
    ("mode", 1.0), ("mode", "gate"), ("mode", "loop"), ("mode", "bogus"), ("mode", "trigger"),
    ("startOffset", "x"), ("startOffset", -1.0), ("startOffset", -0.5), ("startOffset", 12.7), ("startOffset", True),
    ("stopOffset", -3.0), ("stopOffset", 4.0), ("stopOffset", None), ("anything", 1.0),
]
EXPECTED_CODES = [5, 6, 0, 0, 5, 5, 0, 0, 0, 0, 5, 6, 0, 0, 5, 6, 0, 5, 0]
_golden = {}


def golden(key):
    if not _golden:
        _golden.update(np.load(os.path.join(GOLDEN, "reference_sample.npz")))
    return _golden[key]


def cpu_voices(sc):
    """The voices the CPU suite checks (all but the 4096-voice scenario's, of which every 64th)."""
    return list(range(0, sc.n_voices, 64)) if sc.n_voices > 64 else list(range(sc.n_voices))


def _sample_graph():
    return el.render(el.sample({"key": "smp"}, el.in_(0), el.in_(1)))


def reference_prop_codes():
    o = orc.RefRuntime(SR, BS)
    assert o.add_shared_resource("len7", np.arange(7, dtype=np.float32))
    assert o.apply(_sample_graph()) == 0
    sid = el.sample({"key": "smp"}, el.in_(0), el.in_(1)).id()
    return [o.apply([[3, sid, k, v]]) for k, v in PROP_CASES]


def _program_ops(words):
    ops, pc = [], 0
    while pc < len(words):
        w0 = int(words[pc])
        op = w0 & 0xFF
        if op == OP_END:
            break
        ops.append((op, w0 >> 24, [int(x) for x in words[pc + 8:pc + 8 + ((w0 >> 8) & 0xFF)]], int(words[pc + 6])))
        pc += 8 + ((w0 >> 8) & 0xFF)
    return ops


def test_prop_return_codes_match_the_reference():
    rt = Runtime(SR, BS, 4, device=-1)
    assert rt.add_shared_resource("len7", np.arange(7, dtype=np.float32))
    assert rt.apply_instructions(_sample_graph()) == 0
    sid = el.sample({"key": "smp"}, el.in_(0), el.in_(1)).id()
    got = [rt.apply_instructions([[3, sid, k, v]]) for k, v in PROP_CASES]
    ref = reference_prop_codes() if orc.ref_available() else json.loads(str(golden("prop_codes")))
    assert ref == EXPECTED_CODES
    assert got == ref, list(zip(PROP_CASES, got, ref))


def test_sampleseq_and_multichannel_types_stay_unknown():
    rt = Runtime(SR, BS, 2, device=-1)
    for t in ("sampleseq", "sampleseq2", "mc.sample"):
        assert rt.apply_instructions([[0, 5, t]]) == 1, t
    assert rt.apply_instructions([[0, 6, "sample"]]) == 0


@pytest.mark.parametrize("mode,code", [("trigger", 0), ("gate", 1), ("loop", 2)])
@pytest.mark.parametrize("rate", ["input", "none", "nochild"])
def test_program_encodes_the_op(mode, code, rate):
    sc = sample_common.Scenario("plan", mode=mode, rate=rate, n_voices=8)
    rt = Runtime(SR, BS, 8, device=-1)
    sc.setup_gpu(rt)
    ops = _program_ops(rt.program_words(0))
    sample_ops = [o for o in ops if o[0] == OP_SAMPLE]
    if rate == "nochild":                               # no trigger: zeros, no state touched (Sample.h:101-103)
        assert not sample_ops and ops[0][0] == OP_SEG
        return
    assert len(sample_ops) == 1
    op, m, operands, count = sample_ops[0]
    n_children = 2 if rate == "input" else 1
    assert m == code | (4 if n_children == 2 else 0)
    assert count == n_children + 5                      # children, then the five per-voice parameter rows
    assert all(w >> 30 == 1 for w in operands[n_children:n_children + 5])
    # mode is baked into the program: a new mode recompiles at the next block
    other = "loop" if mode != "loop" else "gate"
    assert rt.apply_instructions([[3, sc.sid, "mode", other]]) == 0
    rt.set_option("plan_dry_run", 1)                    # the host side of a block, no rendering
    rt.enqueue_block(sc.n_in, 1, BS)
    (_, m2, _, _), = [o for o in _program_ops(rt.program_words(0)) if o[0] == OP_SAMPLE]
    assert m2 & 3 == {"loop": 2, "gate": 1}[other]


def test_offsets_alone_do_not_cut_the_voice_group_but_a_path_does():
    sc = sample_common.Scenario("plan", n_voices=40)
    rt = Runtime(SR, BS, 40, device=-1)
    sc.setup_gpu(rt)
    assert rt.apply_instructions([[3, sc.sid, "startOffset", 5.0], [3, sc.sid, "stopOffset", 2.0]], (3, 7)) == 0
    assert len(rt.describe()["groups"]) == 1
    assert rt.apply_instructions([[3, sc.sid, "startOffset", -1.0]], (3, 7)) == 6
    assert len(rt.describe()["groups"]) == 1
    assert rt.apply_instructions([[3, sc.sid, "path", "len7"]], (8, 16)) == 0
    assert len(rt.describe()["groups"]) == 3


def test_per_voice_entry_points_check_everything_first():
    sc = sample_common.Scenario("plan", n_voices=16)
    rt = Runtime(SR, BS, 16, device=-1)
    sc.setup_gpu(rt)
    before = rt.snapshot(0)
    sid = sc.sid
    # set_path_per_voice: a bad name, an index out of range, a node that is not per-voice capable
    assert rt.set_path_per_voice(sid, ["len7", "nope"], [0, 1, 0]) == 6
    assert rt.set_path_per_voice(sid, ["len7"], [0, 1]) == -2
    assert rt.set_path_per_voice(sid, ["len7"], [0] * 17) == -2
    assert rt.set_path_per_voice(123456, ["len7"], [0]) == 2
    assert rt.snapshot(0) == before
    # set_property_per_voice: one negative offset anywhere fails the whole call; unknown keys are not per-voice capable
    assert rt.set_property_per_voice(sid, "startOffset", [1.0, 2.0, -1.0, 3.0]) == 6
    assert rt.set_property_per_voice(sid, "stopOffset", [0.0, -7.0]) == 6
    assert rt.set_property_per_voice(sid, "mode", [1.0]) == 5
    assert rt.set_property_per_voice(sid, "seed", [1.0]) == 5
    assert rt.snapshot(0) == before
    # table nodes keep a single path
    t = el.table({"key": "tab", "path": "len7"}, el.const(0.5, key="tpos"))
    assert rt.apply_instructions(el.render(t)) == 0
    assert rt.set_path_per_voice(t.id(), ["len7"], [0] * 16) == 5
    # the successful calls
    assert rt.set_path_per_voice(sid, ["len13", "len7"], [0, 1, 1], 13) == 0
    assert rt.set_property_per_voice(sid, "stopOffset", [2.0, 3.0], 14) == 0
    snap = rt.snapshot(15)
    node = snap[f"0x{sid:08x}"]
    assert node["path"] == "len7" and node["stopOffset"] == 3.0
    assert len(rt.describe()["groups"]) == 1


def test_resources_a_voice_plays_survive_pruning():
    sc = sample_common.Scenario("plan", n_voices=8)
    rt = Runtime(SR, BS, 8, device=-1)
    sc.setup_gpu(rt)
    assert rt.set_path_per_voice(sc.sid, ["len1", "len3001"], [0, 1, 0, 1, 0, 1, 0, 1]) == 0
    rt.prune_shared_resources()
    assert set(rt.get_shared_resource_map_keys()) == {"len1", "len3001"}
    assert rt.set_path_per_voice(sc.sid, ["len1"], [0] * 8) == 0
    rt.prune_shared_resources()
    assert set(rt.get_shared_resource_map_keys()) == {"len1"}


def test_the_warp_pipeline_leaves_sample_programs_whole():
    """The pipeline cut puts values between stages into ring slots, which the out-of-line op bodies do not read: a one-voice
    program with `sample` stays in one piece, the same program without it is cut."""
    names = ["len7"]
    for sampler, want in ((True, 1), (False, 3)):
        rt = Runtime(SR, BS, 6, device=-1, pipeline_stages=3)
        assert rt.add_shared_resource("len7", np.arange(7, dtype=np.float32))
        for v in range(6):
            assert rt.apply_instructions(el.render(sample_common.one_voice_graph(v, names, sampler)), (v, v + 1)) == 0
        assert [g.get("pipeline_stages", 1) for g in rt.describe()["groups"]] == [want] * 6


SCENARIOS = {sc.name: sc for sc in sample_common.scenarios() + [sample_common.many_voices()]}


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_model_matches_the_reference(name):
    """Every checked voice of every GPU scenario: SampleModel bit for bit against the compiled reference, up to the first read
    outside the buffer where a scenario leaves the reference's domain (after it the model gives 0 from that reader, DESIGN.md
    section 4)."""
    sc = SCENARIOS[name]
    voices = cpu_voices(sc)
    model, inputs = sc.model()
    model = model[voices]
    for i, v in enumerate(voices):                      # the reference stops before its first read outside the buffer
        limit = sc.ref_prefix(inputs, v)
        if limit is not None:
            model[i, :, limit:] = np.nan
    if orc.ref_available():
        ref, _ = sc.reference(voices=voices, inputs=inputs)
        assert np.array_equal(model, ref, equal_nan=True), np.argwhere(~((model == ref) | (np.isnan(model) & np.isnan(ref))))[:3]
    want = golden("digest_" + name)
    got = np.array([sample_common.digest(m) for m in model])
    assert (got == want).all(), f"voices {np.array(voices)[got != want][:8]} differ from the stored reference"
    if not sc.ood:
        assert not np.isnan(model).any()
