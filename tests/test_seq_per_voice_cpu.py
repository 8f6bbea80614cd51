"""Per-voice sequences of seq, seq2, sparseq and sparseq2 (Runtime.set_seq_per_voice) on plan-only runtimes: every return code, with
snapshot() and describe() unchanged after a failed call; the per-sequence codes against what [3, id, "seq", v] returns on the same
node (and against the compiled reference where oracle/_ref is built); one voice group after calls that address single voices inside
one tile; and the render program: mode bit 3 and four per-voice parameter operands on the addressed node, the same words as before
for a node never addressed."""
import json

import pytest

from elementary_b200 import Runtime, el
from elementary_b200.runtime import FLAG_MIX
from oracle import oracle as orc

SR, BS = 48000.0, 512
KINDS = ("seq", "seq2", "sparseq", "sparseq2")
GOOD = {
    "seq": [[1.0, 2.0, 3.0], [4.0], []],
    "seq2": [[0.5, -1.5], [7.0, 7.0, 8.0], []],
    "sparseq": [[{"tickTime": 0, "value": 1.0}, {"tickTime": 4, "value": 2.0}], [{"tickTime": 2, "value": 3.0}], []],
    "sparseq2": [[{"time": 0.0, "value": 1.0}, {"time": 0.01, "value": 2.0}], [{"time": 0.005, "value": -1.0}], []],
}
# values a `seq` property may carry, well-formed or not, for every node kind
VALUES = [[1.0, 2.0], [], "text", 3.0, None, True, {"a": 1}, [1.0, "x"], [[1.0]], [{"tickTime": 0, "value": 1.0}],
          [{"tickTime": 0}], [{"value": 1.0}], [{"time": 0.5, "value": 2.0}], [{"time": "0", "value": 2.0}],
          [{"tickTime": 1, "value": 1.0}, 2.0], [1.0, {"time": 0.0, "value": 1.0}]]


def seq_node(kind, key, value):
    """The node fed by host inputs only, so that its program holds no parameter operand of its own."""
    if kind == "sparseq2":
        return el.sparseq2({"seq": value, "key": key}, el.in_(0))
    return getattr(el, kind)({"seq": value, "key": key}, el.in_(0), el.in_(1))


def runtime(kind, n_voices=45, extra=(), **opts):
    rt = Runtime(SR, BS, n_voices, device=-1, plan_dry_run=1, **opts)
    a, b = seq_node(kind, "a", GOOD[kind][0]), seq_node(kind, "b", GOOD[kind][1])
    assert rt.apply_instructions(el.render(a, b, *extra)) == 0, rt.last_error()
    return rt, a.id(), b.id()


def state(rt):
    return rt.describe()["groups"], [rt.snapshot(v) for v in range(rt.num_voices)], rt.program_words(0).tolist()


def ops(rt):
    """(header, operand words) of each op up to OP_END, in the program the next block renders with."""
    rt.enqueue_block(0, 1, BS, flags=FLAG_MIX)
    w = [int(x) for x in rt.program_words(0)]
    out, pc = [], 0
    while pc + 8 <= len(w):
        n = (w[pc] >> 8) & 0xFF
        out.append((w[pc:pc + 8], w[pc + 8:pc + 8 + n]))
        if (w[pc] & 0xFF) == 0:
            break
        pc += 8 + n
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_return_codes_and_failed_calls_change_nothing(kind):
    other = el.const(0.5, key="c")
    rt, aid, _ = runtime(kind, extra=(el.mul(other, el.in_(2)),), tile_width=8)
    seqs = GOOD[kind]
    before = state(rt)
    for args, code in [
        ((aid, seqs, [0, 1], 44), -2),                  # voice range past the end
        ((aid, seqs, [0], -1), -2),
        ((aid, seqs, [0, 3], 0), -2),                   # index outside [0, numSeqs)
        ((aid, seqs, [-1, 0], 0), -2),
        ((123456, seqs, [0, 1], 0), 2),                 # NodeNotFound
        ((other.id(), seqs, [0, 1], 0), 5),             # InvalidPropertyType: not a sequencer
        ((aid, seqs + ["text"], [0, 1], 0), 5),         # a non-array, even one no voice takes
        ((aid, seqs + [[{"x": 1}, 2]], [0], 0), 8),     # a malformed entry
        ((aid, seqs + [b"[1, 2"], [0], 0), 8),          # not JSON
    ]:
        assert rt.set_seq_per_voice(args[0], args[1], args[2], voice_begin=args[3]) == code, (args, rt.last_error())
        assert state(rt) == before, args
    assert rt.set_seq_per_voice(aid, seqs, []) == 0   # nothing to do
    assert state(rt) == before


@pytest.mark.parametrize("kind", KINDS)
def test_node_missing_in_one_group_of_the_range(kind):
    rt = Runtime(SR, BS, 8, device=-1)
    node = seq_node(kind, "a", GOOD[kind][0])
    assert rt.apply_instructions(el.render(node), voices=(0, 4)) == 0
    assert rt.apply_instructions(el.render(el.cycle(220.0)), voices=(4, 8)) == 0
    before = state(rt)
    assert rt.set_seq_per_voice(node.id(), GOOD[kind], [1] * 8) == 2
    assert state(rt) == before
    assert rt.set_seq_per_voice(node.id(), GOOD[kind], [1] * 4) == 0


@pytest.mark.parametrize("kind", KINDS)
def test_per_seq_codes_match_json_seq(kind):
    """Each value gives the code [3, id, "seq", value] gives on the same node — and, where oracle/_ref is built, the reference."""
    for value in VALUES:
        rt, aid, _ = runtime(kind, n_voices=4)
        twin, tid, _ = runtime(kind, n_voices=4)
        want = twin.apply_instructions([[3, tid, "seq", value]])
        before = state(rt)
        got = rt.set_seq_per_voice(aid, [GOOD[kind][0], value], [0, 0, 0, 0])
        assert got == want, (value, got, want)
        if got != 0:
            assert state(rt) == before, value
        if orc.ref_available():
            o = orc.RefRuntime(SR, BS)
            assert o.apply(el.render(seq_node(kind, "a", GOOD[kind][0]), seq_node(kind, "b", GOOD[kind][1]))) == 0
            assert o.apply([[3, aid, "seq", value]]) == want, value


@pytest.mark.parametrize("kind", KINDS)
def test_single_voices_inside_one_tile_keep_one_group(kind):
    rt, aid, _ = runtime(kind, tile_width=8)
    for v in (0, 3, 5, 17, 44):
        assert rt.set_seq_per_voice(aid, GOOD[kind], [v % 3], voice_begin=v) == 0, rt.last_error()
    assert len(rt.describe()["groups"]) == 1
    # what the same sequences cost through JSON on voice sub-ranges: cuts on tile boundaries are refused inside a tile
    assert rt.apply_instructions([[3, aid, "seq", GOOD[kind][1]]], voices=(3, 4)) == 7
    assert len(rt.describe()["groups"]) == 1


@pytest.mark.parametrize("kind", KINDS)
def test_program_words(kind):
    rt, aid, bid = runtime(kind, tile_width=4)
    before = ops(rt)
    assert rt.set_seq_per_voice(aid, GOOD[kind], [v % 3 for v in range(45)]) == 0, rt.last_error()
    after = ops(rt)
    assert len(after) == len(before)
    changed = [i for i, (x, y) in enumerate(zip(before, after)) if x != y]
    seg = [i for i in changed if (before[i][0][0] & 0xFF) == 1]       # OP_SEG: its skip count (w3) covers the longer op
    for i in seg:
        (h0, _), (h1, _) = before[i], after[i]
        assert h1[:3] + h1[4:] == h0[:3] + h0[4:] and h1[3] == h0[3] + 4
    seqop = [i for i in changed if i not in seg]
    assert len(seqop) == 1, changed                         # only the addressed node's op; node b keeps its words
    (h0, o0), (h1, o1) = before[seqop[0]], after[seqop[0]]
    assert (h0[0] & 0xFF) == (h1[0] & 0xFF) and h1[1] == h0[1]
    assert (h0[0] >> 24) & 8 == 0 and (h1[0] >> 24) == ((h0[0] >> 24) | 8)
    assert h1[6] == h0[6] + 4                               # four more operands
    assert h1[4] == h1[5] == 0 and h1[2] == 0               # the group's pointer and count are not read
    assert h0[4] | h0[5] != 0
    n_in = h0[6]
    rows = o1[n_in:n_in + 4]
    assert o1[:n_in] == o0[:n_in]                           # the inputs, then the rows, then the immediates
    assert all(w >> 30 == 1 for w in rows) and len(set(rows)) == 4                        # K_PARAM operands
    if kind != "sparseq2":                                  # the first immediate: the offset (sparseq2's is the unread generation)
        assert o1[n_in + 4] == o0[n_in]
    changed = seqop
    # later calls only write rows; a whole-group JSON `seq` keeps the per-voice form
    assert rt.set_seq_per_voice(aid, GOOD[kind], [1], voice_begin=7) == 0
    assert ops(rt)[changed[0]][0][:3] == h1[:3]
    assert rt.apply_instructions([[3, aid, "seq", GOOD[kind][1]]]) == 0
    assert (ops(rt)[changed[0]][0][0] >> 24) & 8


@pytest.mark.parametrize("kind", KINDS)
def test_snapshot_reports_the_highest_addressed_voice(kind):
    rt, aid, _ = runtime(kind, tile_width=8)
    key = f"0x{aid & 0xFFFFFFFF:08x}"
    assert rt.set_seq_per_voice(aid, GOOD[kind], [2, 1, 0, 1], voice_begin=10) == 0
    assert json.loads(json.dumps(rt.snapshot(0)[key]["seq"])) == GOOD[kind][1]
    assert rt.set_seq_per_voice(aid, GOOD[kind], [2]) == 0
    assert rt.snapshot(0)[key]["seq"] == GOOD[kind][2]


def test_empty_sequences_everywhere_emit_zeros():
    """seq / seq2 / sparseq2: the op is emitted while any voice has a sequence, and becomes zeros when none has."""
    for kind in ("seq", "seq2", "sparseq2"):
        rt, aid, _ = runtime(kind, n_voices=6)
        n_ops = len(ops(rt))
        assert rt.set_seq_per_voice(aid, GOOD[kind], [2, 2, 2, 2, 2, 0]) == 0
        assert any((h[0] >> 24) & 8 for h, _ in ops(rt))
        assert rt.set_seq_per_voice(aid, GOOD[kind], [2], voice_begin=5) == 0
        assert not any((h[0] >> 24) & 8 for h, _ in ops(rt))
        assert len(ops(rt)) == n_ops
