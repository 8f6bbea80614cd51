"""Records tests/golden/per_voice_program_words.json: what the per-voice setters leave behind on plan-only engines.  For a `sample`
graph and for each of seq, seq2, sparseq and sparseq2 at three tile widths, a fixed script of per-voice calls (path, sample offsets,
const values and tables, sequences, among them the first set_seq_per_voice of a node, which allocates its rows), JSON `seq` batches
after per-voice calls, and a voice-group cut between them.  After every step it records the masked program words of every voice
group, describe()["groups"] and snapshot() of every voice.  tests/test_per_voice_setters_cpu.py replays the script against it.

    python tests/golden/make_per_voice_program_words.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)                                        # make_program_words
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))      # the repository: elementary_b200

from make_program_words import masked  # noqa: E402

SR, BS, VOICES, CUT = 48000.0, 512, 64, 32   # the cut is a tile boundary at every width
WIDTHS = (1, 4, 32)
KINDS = ("sample", "seq", "seq2", "sparseq", "sparseq2")
SEQS = {
    "seq": [[1.0, 2.0, 3.0], [4.0], []],
    "seq2": [[0.5, -1.5], [7.0, 7.0, 8.0], []],
    "sparseq": [[{"tickTime": 0, "value": 1.0}, {"tickTime": 4, "value": 2.0}], [{"tickTime": 2, "value": 3.0}], []],
    "sparseq2": [[{"time": 0.0, "value": 1.0}, {"time": 0.01, "value": 2.0}], [{"time": 0.005, "value": -1.0}], []],
}
RESOURCES = {"len7": np.arange(7, dtype=np.float32), "len12": np.linspace(-1.0, 1.0, 12).astype(np.float32)}


def graph(kind):
    """(batch, id of node a, id of node b, id of the const): two per-voice capable nodes of the kind and one const."""
    from elementary_b200 import el
    c = el.const(0.5, key="c")
    if kind == "sample":
        a = el.sample({"key": "a", "path": "len7"}, el.in_(0), el.in_(1))
        b = el.sample({"key": "b"}, el.in_(0))
    elif kind == "sparseq2":
        a, b = (el.sparseq2({"seq": SEQS[kind][k], "key": key}, el.in_(0)) for k, key in ((0, "a"), (1, "b")))
    else:
        a, b = (getattr(el, kind)({"seq": SEQS[kind][k], "key": key}, el.in_(0), el.in_(1)) for k, key in ((0, "a"), (1, "b")))
    return el.render(a, b, el.mul(c, el.in_(2))), a.id(), b.id(), c.id()


def runtime(kind, L):
    from elementary_b200 import Runtime
    rt = Runtime(SR, BS, VOICES, device=-1, plan_dry_run=1, tile_width=L)
    for name, data in RESOURCES.items():
        assert rt.add_shared_resource(name, data)
    batch, aid, bid, cid = graph(kind)
    assert rt.apply_instructions(batch) == 0, rt.last_error()
    return rt, aid, bid, cid


def steps(kind, aid, bid, cid):
    """The script: (name, call(rt) -> return code), each expected to return 0."""
    idx = lambda n, k: [(7 * i + 3) % k for i in range(n)]   # noqa: E731
    const = [
        ("const per voice", lambda rt: rt.set_property_per_voice(cid, "value", np.arange(10) * 0.25, voice_begin=3)),
        ("const table", lambda rt: rt.set_const_table([cid], np.arange(20, dtype=np.float32).reshape(1, 20) - 4.0, voice_begin=24)),
    ]
    if kind == "sample":
        names = ["len7", "len12"]
        script = [
            ("path per voice", lambda rt: rt.set_path_per_voice(aid, names, idx(9, 2), voice_begin=2)),
            ("startOffset per voice", lambda rt: rt.set_property_per_voice(aid, "startOffset", np.arange(6) + 1.5, voice_begin=4)),
            ("stopOffset per voice", lambda rt: rt.set_property_per_voice(bid, "stopOffset", [3.0, 0.0, 9.0], voice_begin=60)),
            ("JSON startOffset", lambda rt: rt.apply_instructions([[3, aid, "startOffset", 2.0]], voices=(8, 12))),
            ("cut", lambda rt: rt.apply_instructions([[3, aid, "mode", "loop"]], voices=(CUT, VOICES))),
            ("path across the cut", lambda rt: rt.set_path_per_voice(bid, names[::-1], idx(24, 2), voice_begin=20)),
            ("JSON path after per-voice", lambda rt: rt.apply_instructions([[3, aid, "path", "len12"]], voices=(CUT, VOICES))),
            ("offsets across the cut", lambda rt: rt.set_property_per_voice(aid, "stopOffset", np.arange(16) * 0.5, voice_begin=24)),
        ]
    else:
        seqs = SEQS[kind]
        script = [
            ("first seq per voice", lambda rt: rt.set_seq_per_voice(aid, seqs, idx(9, 3), voice_begin=2)),
            ("seq per voice again", lambda rt: rt.set_seq_per_voice(aid, seqs[::-1], idx(3, 3), voice_begin=5)),
            ("JSON seq after per-voice", lambda rt: rt.apply_instructions([[3, aid, "seq", seqs[1]]])),
            ("cut", lambda rt: rt.apply_instructions([[3, bid, "seq", seqs[0]]], voices=(CUT, VOICES))),
            ("seq across the cut", lambda rt: rt.set_seq_per_voice(aid, seqs, idx(24, 3), voice_begin=20)),
            ("first seq per voice, second group", lambda rt: rt.set_seq_per_voice(bid, seqs, idx(5, 3), voice_begin=40)),
            ("JSON seq in one group", lambda rt: rt.apply_instructions([[3, aid, "seq", seqs[0]]], voices=(CUT, VOICES))),
        ]
    return script[:3] + const + script[3:]


def state(rt):
    """Masked program words of every voice group (the program the next block renders with), describe()["groups"], and every voice's
    snapshot(), as the distinct snapshots and the index of each voice's among them."""
    from elementary_b200.runtime import FLAG_MIX
    rt.enqueue_block(0, 1, BS, flags=FLAG_MIX)
    groups = rt.describe()["groups"]
    snaps, voice_snap = [], []
    for v in range(VOICES):
        s = rt.snapshot(v)
        if s not in snaps:
            snaps.append(s)
        voice_snap.append(snaps.index(s))
    return {"programs": [masked(rt.program_words(g["v0"])) for g in groups], "groups": groups,
            "snapshots": snaps, "voice_snapshot": voice_snap}


def replay(kind, L):
    rt, aid, bid, cid = runtime(kind, L)
    out = [{"step": "graph", **state(rt)}]
    for name, call in steps(kind, aid, bid, cid):
        assert call(rt) == 0, (kind, L, name, rt.last_error())
        out.append({"step": name, **state(rt)})
    return out


def record():
    return {f"{kind}/L{L}": replay(kind, L) for kind in KINDS for L in WIDTHS}


if __name__ == "__main__":
    with open(os.path.join(HERE, "per_voice_program_words.json"), "w") as f:
        json.dump(record(), f, separators=(",", ":"), sort_keys=True)
