"""Per-voice impulse responses of `convolve` (Runtime.set_path_per_voice) on plan-only runtimes: return codes, all-or-nothing
application, one voice group however many IRs, the IR spectra bank and the snapshot rule."""
import numpy as np

from elementary_b200 import Runtime, el, graphs

SR, BS = 48000.0, 512


def plan(n_voices):
    return Runtime(SR, BS, n_voices, device=-1)


def irs(k, taps=1500):
    base = np.asarray(graphs.lcg_ir(taps), dtype=np.float32)
    return {f"ir{i}": base * (1.0 + 0.1 * i) for i in range(k)}


def conv_runtime(n_voices, k=7, path="ir0", wrap=None):
    rt = plan(n_voices)
    for name, data in irs(k).items():
        assert rt.add_shared_resource(name, data)
    cv = el.convolve({"path": path, "key": "cv"}, el.in_(0))
    rt.renderer = el.Renderer()
    assert rt.apply_instructions(rt.renderer.render(wrap(cv) if wrap else cv)) == 0, rt.last_error()
    return rt, cv.id()


def convolvers(rt):
    return [c for g in rt.describe()["groups"] for c in g.get("convolvers", [])]


def test_error_codes():
    rt, cid = conv_runtime(8, wrap=lambda cv: el.mul(el.const(0.5, key="c"), cv))
    names = ["ir0", "ir1"]
    assert rt.set_path_per_voice(cid, names, [0, 1], voice_begin=7) == -2         # voice range past the end
    assert rt.set_path_per_voice(cid, names, [0, 1], voice_begin=-1) == -2
    assert rt.set_path_per_voice(cid, names, [0, 2]) == -2                        # index outside [0, numNames)
    assert rt.set_path_per_voice(cid, names, [-1, 0]) == -2
    assert rt.set_path_per_voice(123456, names, [0, 1]) == 2                      # NodeNotFound
    other = el.const(0.5, key="c").id()
    assert rt.set_path_per_voice(other, names, [0, 1]) == 5                       # InvalidPropertyType: not a convolve
    assert "per-voice" in rt.last_error()
    assert rt.set_path_per_voice(cid, ["ir0", "nope"], [0, 1]) == 6               # InvalidPropertyValue: no such resource
    assert rt.set_path_per_voice(cid, names, []) == 0                             # nothing to do


def test_node_missing_in_one_group_of_the_range():
    rt = plan(8)
    for name, data in irs(2).items():
        assert rt.add_shared_resource(name, data)
    cv = el.convolve({"path": "ir0", "key": "cv"}, el.in_(0))
    cid = cv.id()
    assert rt.apply_instructions(el.render(cv), voices=(0, 4)) == 0
    assert rt.apply_instructions(el.render(el.cycle(220.0)), voices=(4, 8)) == 0  # voices 4..7: another graph, without the node
    assert len(rt.describe()["groups"]) == 2
    assert rt.set_path_per_voice(cid, ["ir1"], [0] * 8) == 2
    assert convolvers(rt)[0]["irs"] == 1                                          # nothing changed in the first group
    assert rt.set_path_per_voice(cid, ["ir1"], [0] * 4) == 0


def test_failed_call_changes_nothing():
    rt, cid = conv_runtime(6)
    before = (rt.describe(), rt.snapshot())
    names = ["ir1", "ir2", "ir3", "ir4", "missing", "ir5"]                       # the 5th of 6 names is unknown
    assert rt.set_path_per_voice(cid, names, [0, 1, 2, 3, 5, 5]) == 6
    assert (rt.describe(), rt.snapshot()) == before
    assert convolvers(rt)[0]["irs"] == 1 and convolvers(rt)[0]["form"] == "shared"


def test_37_voices_7_irs_stay_one_group():
    rt, cid = conv_runtime(37)
    names = [f"ir{i}" for i in range(7)]
    idx = [(v * 3) % 7 for v in range(37)]
    assert rt.set_path_per_voice(cid, names, idx) == 0, rt.last_error()
    d = rt.describe()
    assert len(d["groups"]) == 1
    c = convolvers(rt)
    assert len(c) == 1 and c[0]["irs"] == 7 and c[0]["form"] == "per_channel" and c[0]["partitions"] == 3
    assert d["ir_bank"] == 7
    # a sub-range: still one group
    assert rt.set_path_per_voice(cid, names, [6, 5, 4], voice_begin=10) == 0
    assert len(rt.describe()["groups"]) == 1


def test_bank_computes_one_spectrum_set_per_resource():
    rt, cid = conv_runtime(1000, k=3)
    assert rt.describe()["ir_bank"] == 1                                          # the JSON path on every voice: one entry
    assert rt.set_path_per_voice(cid, ["ir1"], [0] * 1000) == 0
    assert rt.describe()["ir_bank"] == 1                                          # ir0 is used by nobody any more
    c = convolvers(rt)[0]
    assert c["irs"] == 1 and c["form"] == "shared"
    assert rt.set_path_per_voice(cid, ["ir1", "ir2"], [v % 2 for v in range(500)], voice_begin=500) == 0
    assert rt.describe()["ir_bank"] == 2 and convolvers(rt)[0]["irs"] == 2
    # a second convolver on the same resource shares the entry
    rt2 = plan(4)
    for name, data in irs(3).items():
        rt2.add_shared_resource(name, data)
    g = el.convolve({"path": "ir1", "key": "b"}, el.convolve({"path": "ir1", "key": "a"}, el.in_(0)))
    assert rt2.apply_instructions(el.render(g)) == 0
    assert rt2.describe()["ir_bank"] == 1 and len(convolvers(rt2)) == 2


def test_snapshot_reports_the_highest_addressed_voice():
    rt, cid = conv_runtime(8)
    key = "0x%08x" % (cid & 0xFFFFFFFF)
    assert rt.snapshot()[key]["path"] == "ir0"
    assert rt.set_path_per_voice(cid, ["ir3", "ir5", "ir2"], [1, 0, 2, 1], voice_begin=2) == 0
    assert rt.snapshot()[key]["path"] == "ir5"                                    # voice 5 got names[index[3]]
    assert rt.set_path_per_voice(cid, ["ir6"], [0], voice_begin=0) == 0
    assert rt.snapshot()[key]["path"] == "ir6"


def test_convolver_without_path_gets_per_voice_irs():
    rt = plan(4)
    for name, data in irs(2).items():
        rt.add_shared_resource(name, data)
    cv = el.convolve({"key": "cv"}, el.in_(0))
    assert rt.apply_instructions(el.render(cv)) == 0
    assert rt.set_path_per_voice(cv.id(), ["ir0", "ir1"], [0, 1], voice_begin=1) == 0
    c = convolvers(rt)[0]
    assert c["irs"] == 3 and c["form"] == "per_channel"                           # voices 0 and 3 have no IR (silence)


def test_whole_group_json_path_restores_the_shared_form_and_cuts_keep_irs():
    rt, cid = conv_runtime(64)
    assert rt.set_path_per_voice(cid, ["ir1", "ir2"], [v % 2 for v in range(64)]) == 0
    assert convolvers(rt)[0]["form"] == "per_channel"
    # a structural batch on a sub-range cuts the group: both halves keep their voices' IRs
    assert rt.apply_instructions(rt.renderer.render(el.mul(0.5, el.convolve({"path": "ir0", "key": "cv"}, el.in_(0)))), voices=(32, 64)) == 0
    groups = rt.describe()["groups"]
    assert len(groups) == 2 and all(g["convolvers"][0]["irs"] == 2 for g in groups)
    rt2, cid2 = conv_runtime(8)
    assert rt2.set_path_per_voice(cid2, ["ir1", "ir2"], [0, 1], voice_begin=3) == 0
    assert convolvers(rt2)[0]["irs"] == 3
    # `path` through JSON on the whole group: a fresh shared-IR convolver at the commit
    assert rt2.apply_instructions(rt2.renderer.render(el.convolve({"path": "ir4", "key": "cv"}, el.in_(0)))) == 0
    c = convolvers(rt2)
    assert len(rt2.describe()["groups"]) == 1 and c[0]["irs"] == 1 and c[0]["form"] == "shared"


def test_abi_exports_the_entry_point():
    from elementary_b200.runtime import load_library
    assert hasattr(load_library(), "elem_b200_set_path_per_voice")


def test_seeded_lcg_ir_keeps_the_default_sequence():
    import math
    s, want = 1, []
    for n in range(1000):
        s = (s * 1664525 + 1013904223) & 0xFFFFFFFF
        want.append(((s >> 8) / float(1 << 24) - 0.5) * 0.01 * math.exp(-6.0 * n / 1000))
    assert graphs.lcg_ir(1000) == want == graphs.lcg_ir(1000, seed=1)
    assert graphs.lcg_ir(1000, seed=2) != want
