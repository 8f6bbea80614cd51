"""GPU: per-voice impulse responses of `convolve` (Runtime.set_path_per_voice) — one voice group, one K3 launch per chunk, each
voice against the compiled reference ConvolutionNode with that voice's `path` (tolerance as tests/test_convolve_gpu.py: 1e-5 of
the peak), and the exactness the per-channel form promises: a channel's bits equal the shared-IR form's on the same IR and input."""
import numpy as np
import pytest

from elementary_b200 import Runtime, el, graphs
from helpers import oracle_cls, oracle_render

pytestmark = pytest.mark.gpu
SR = 48000.0
BASE = np.asarray(graphs.lcg_ir(16384), dtype=np.float32)


def check(got, ref, tol=1e-5):
    peak = np.abs(ref).max()
    err = np.abs(got.astype(np.float64) - ref.astype(np.float64)).max()
    assert peak > 0 and err <= tol * peak, f"max err {err:.3g} vs peak {peak:.3g} (ratio {err / peak:.3g})"


def noise(n_voices, n, seed=1):
    return np.random.default_rng(seed).uniform(-0.25, 0.25, size=(n_voices, 1, n)).astype(np.float32)


def seven_irs():
    """1, 300, 512, 513, 4097 and 16384 taps, and one that trims to nothing."""
    out = {f"t{t}": BASE[:t] * (3.0 + 0.25 * k) for k, t in enumerate([1, 300, 512, 513, 4097, 16384])}
    out["zero"] = np.zeros(64, dtype=np.float32)
    return out


def runtime(n_voices, resources, path, bs=512, wrap=None, **opts):
    rt = Runtime(SR, bs, n_voices, device=0, **opts)
    for k, v in resources.items():
        assert rt.add_shared_resource(k, v)
    cv = el.convolve({"path": path, "key": "cv"}, el.in_(0))
    batch = el.render(wrap(cv) if wrap else cv)
    assert rt.apply_instructions(batch) == 0, rt.last_error()
    return rt, cv.id(), batch


def reference(batch, cid, names_v, resources, x, n_blocks, bs=512):
    return oracle_render(batch, n_blocks, 1, SR, bs, x, voice_batches=[[[3, cid, "path", nm]] for nm in names_v], resources=resources)


def convolvers(rt):
    return [c for g in rt.describe()["groups"] for c in g.get("convolvers", [])]


def launches_per_block(rt, x, n_blocks=4):
    rt.render_voices(1, 1, x[:, :, :rt.block_size])
    l0 = rt.kernel_launches
    rt.render_voices(n_blocks, 1, x[:, :, :n_blocks * rt.block_size])
    return (rt.kernel_launches - l0) / n_blocks


def test_37_voices_7_irs_match_the_reference_in_one_group():
    res = seven_irs()
    names = list(res)
    idx = [(5 * v + 2) % 7 for v in range(37)]
    nb = 40
    rt, cid, batch = runtime(37, res, "t300")
    assert rt.set_path_per_voice(cid, names, idx) == 0, rt.last_error()
    assert len(rt.describe()["groups"]) == 1
    c = convolvers(rt)[0]
    assert c["irs"] == 7 and c["form"] == "per_channel"
    x = noise(37, nb * 512, seed=3)
    got, _ = rt.render_voices(nb, 1, x)
    ref = reference(batch, cid, [names[i] for i in idx], res, x, nb)
    for v in range(37):
        if names[idx[v]] == "zero":
            assert not got[v].any() and not ref[v].any()
        else:
            check(got[v], ref[v])
    single, _, _ = runtime(37, res, "t300")
    assert launches_per_block(rt, x) == launches_per_block(single, x)


def test_same_ir_on_every_voice_is_bit_identical_to_the_json_path():
    res = {"a": BASE[:5000] * 2.0, "b": BASE[:3000]}
    x = noise(9, 12 * 512, seed=5)
    rt, cid, _ = runtime(9, res, "b")
    assert rt.set_path_per_voice(cid, ["a"], [0] * 9) == 0
    assert convolvers(rt)[0]["form"] == "shared"
    js, _, _ = runtime(9, res, "a")
    assert np.array_equal(rt.render_voices(12, 1, x)[0], js.render_voices(12, 1, x)[0])


def test_per_channel_form_is_bit_identical_to_the_shared_form():
    res = {"a": BASE[:5000] * 2.0, "b": BASE[:9000] * 1.5}
    n, nb = 11, 14
    x = noise(n, nb * 512, seed=7)
    idx = [0, 1, 1, 0, 1, 0, 0, 1, 1, 1, 0]
    rt, cid, _ = runtime(n, res, "a")
    assert rt.set_path_per_voice(cid, ["a", "b"], idx) == 0
    assert convolvers(rt)[0]["form"] == "per_channel"
    got = rt.render_voices(nb, 1, x)[0]
    for k, name in enumerate(["a", "b"]):
        single, _, _ = runtime(n, res, name)
        want = single.render_voices(nb, 1, x)[0]
        for v in range(n):
            if idx[v] == k:
                assert np.array_equal(got[v], want[v]), (name, v)


def test_reassigning_a_subset_mid_stream_with_ragged_calls():
    """A subset of voices gets new IRs between ragged calls (including one longer than any before: the ring grows); the other
    voices are bit-identical to a run without the reassignment, the reassigned ones match a reference given the `path` at the same
    call boundary."""
    res = {"a": BASE[:2000] * 2.0, "b": BASE[:1200] * 3.0, "long": BASE[:7000] * 1.5}
    n = 6
    sizes = [512, 100, 37, 375, 1, 512, 512, 300, 212, 512]
    x = noise(n, sum(sizes), seed=11)
    rt, cid, batch = runtime(n, res, "a")
    plain, _, _ = runtime(n, res, "a")
    assert rt.set_path_per_voice(cid, ["a", "b"], [0, 0, 0, 1, 1, 1]) == 0
    assert plain.set_path_per_voice(cid, ["a", "b"], [0, 0, 0, 1, 1, 1]) == 0
    outs, outs_plain, pos = [], [], 0
    cut = 4                                       # before the 5th call: 512 + 100 + 37 + 375 samples in, mid-partition
    for k, m in enumerate(sizes):
        if k == cut:
            assert rt.set_path_per_voice(cid, ["long", "b"], [0, 0, 1, 1], voice_begin=1) == 0   # voices 1..4: long, long, b, b
            assert convolvers(rt)[0]["partitions"] == 14
        outs.append(rt.process_voices(x[:, :, pos:pos + m], 1, m)[0])
        outs_plain.append(plain.process_voices(x[:, :, pos:pos + m], 1, m)[0])
        pos += m
    got, base = np.concatenate(outs, axis=2), np.concatenate(outs_plain, axis=2)
    for v in (0, 5):
        assert np.array_equal(got[v], base[v]), v
    first = {v: ("a" if v < 3 else "b") for v in range(n)}
    later = {1: "long", 2: "long", 3: "b", 4: "b"}
    for v in later:
        o = oracle_cls()(SR, 512)
        for k2, d in res.items():
            assert o.add_shared_resource(k2, d)
        assert o.apply(batch) == 0 and o.apply([[3, cid, "path", first[v]]]) == 0
        parts, p = [], 0
        for k, m in enumerate(sizes):
            if k == cut:
                assert o.apply([[3, cid, "path", later[v]]]) == 0
            parts.append(o.process(x[v, :, p:p + m], 1, m))
            p += m
        check(got[v], np.concatenate(parts, axis=1))


def test_root_epilogue_and_k1_stage_agree():
    res = {"a": BASE[:3000], "b": BASE[:6000] * 2.0}
    n, nb = 7, 10
    x = noise(n, nb * 512, seed=13)
    outs = {}
    for f in (1, 0):
        rt, cid, _ = runtime(n, res, "a", fuse_conv_root=f)
        assert rt.set_path_per_voice(cid, ["a", "b"], [v % 2 for v in range(n)]) == 0
        outs[f] = rt.render_voices(nb, 2, x)
    assert np.array_equal(outs[1][0], outs[0][0]) and np.array_equal(outs[1][1], outs[0][1])
    assert np.abs(outs[1][0][:, 0]).max() > 0 and not outs[1][0][:, 1].any()


def test_dry_wet_graph_two_convolvers_in_series_and_block_sizes():
    res = {"a": BASE[:3000] * 2.0, "b": BASE[:1500] * 4.0, "c": BASE[:600] * 3.0}
    # dry/wet through K1 stages
    xin = el.tanh(el.mul(2.0, el.in_(0)))
    wet = el.convolve({"path": "a", "key": "w"}, xin)
    g = el.add(el.mul(0.7, wet), el.mul(0.3, xin))
    n, nb = 5, 8
    x = noise(n, nb * 512, seed=17)
    rt = Runtime(SR, 512, n, device=0)
    for k, v in res.items():
        rt.add_shared_resource(k, v)
    batch = el.render(g)
    assert rt.apply_instructions(batch) == 0
    names = ["a", "b", "c", "b", "a"]
    assert rt.set_path_per_voice(wet.id(), ["a", "b", "c"], [0, 1, 2, 1, 0]) == 0
    got, _ = rt.render_voices(nb, 1, x)
    check(got, reference(batch, wet.id(), names, res, x, nb))
    # two convolvers in series, each with its own assignment
    a = el.convolve({"path": "a", "key": "s1"}, el.in_(0))
    b = el.convolve({"path": "a", "key": "s2"}, el.mul(0.5, a))
    rt = Runtime(SR, 512, n, device=0)
    for k, v in res.items():
        rt.add_shared_resource(k, v)
    batch = el.render(b)
    assert rt.apply_instructions(batch) == 0
    ia, ib = [0, 1, 2, 0, 1], [2, 2, 0, 1, 1]
    assert rt.set_path_per_voice(a.id(), ["a", "b", "c"], ia) == 0 and rt.set_path_per_voice(b.id(), ["a", "b", "c"], ib) == 0
    got, _ = rt.render_voices(nb, 1, x)
    ref = oracle_render(batch, nb, 1, SR, 512, x, resources=res,
                        voice_batches=[[[3, a.id(), "path", "abc"[ia[v]]], [3, b.id(), "path", "abc"[ib[v]]]] for v in range(n)])
    check(got, ref, tol=2e-5)
    # other block sizes
    for bs in (64, 1024):
        nbs = 3 * 2048 // bs
        xb = noise(3, nbs * bs, seed=bs)
        rt, cid, batch = runtime(3, res, "a", bs=bs)
        assert rt.set_path_per_voice(cid, ["c", "b"], [0, 1], voice_begin=1) == 0
        got, _ = rt.render_voices(nbs, 1, xb)
        check(got, reference(batch, cid, ["a", "c", "b"], res, xb, nbs, bs=bs))


def test_group_cut_after_assignment_continues_bit_identically():
    res = {"a": BASE[:3000] * 2.0, "b": BASE[:5000]}
    n = 64
    x = noise(n, 12 * 512, seed=19)
    outs = []
    for cut in (False, True):
        rt, cid, _ = runtime(n, res, "a", tile_width=1)
        assert rt.set_path_per_voice(cid, ["a", "b"], [(v // 3) % 2 for v in range(n)]) == 0
        o1, _ = rt.render_voices(5, 1, x[:, :, :5 * 512])
        if cut:   # a value-irrelevant structural batch on voices 32..63: the group is cut there
            assert rt.apply_instructions([[0, 777, "const"], [3, 777, "value", 1.0], [5]], voices=(32, 64)) == 0
            assert len(rt.describe()["groups"]) == 2 and all(g["convolvers"][0]["irs"] == 2 for g in rt.describe()["groups"])
        o2, _ = rt.render_voices(7, 1, x[:, :, 5 * 512:])
        outs.append(np.concatenate([o1, o2], axis=2))
    assert np.array_equal(outs[0], outs[1])


def test_whole_group_json_path_brings_back_the_shared_form():
    res = {"a": BASE[:3000] * 2.0, "b": BASE[:5000], "c": BASE[:900] * 3.0}
    n, nb = 6, 10
    x = noise(n, nb * 512, seed=23)
    rt, cid, batch = runtime(n, res, "a")
    assert rt.set_path_per_voice(cid, ["a", "b"], [0, 1, 0, 1, 0, 1]) == 0
    rt.render_voices(3, 1, x[:, :, :3 * 512])
    assert rt.apply_instructions([[3, cid, "path", "c"], [5]]) == 0
    got, _ = rt.render_voices(nb, 1, x)
    c = convolvers(rt)[0]
    assert c["irs"] == 1 and c["form"] == "shared"
    for v in range(n):    # the reference runs the same 3 blocks first: its root has faded in like the engine's
        o = oracle_cls()(SR, 512)
        for k, d in res.items():
            assert o.add_shared_resource(k, d)
        assert o.apply(batch) == 0 and o.apply([[3, cid, "path", "ab"[v % 2]]]) == 0
        o.render(3, 1, 512, x[v, :, :3 * 512])
        assert o.apply([[3, cid, "path", "c"]]) == 0
        check(got[v], o.render(nb, 1, 512, x[v]))


def test_prune_after_assignment_leaves_the_output_unchanged():
    res = {"a": BASE[:3000] * 2.0, "b": BASE[:5000], "c": BASE[:900] * 3.0}
    n, nb = 4, 8
    x = noise(n, nb * 512, seed=29)
    outs = []
    for prune in (False, True):
        rt, cid, _ = runtime(n, res, "a")
        assert rt.set_path_per_voice(cid, ["b", "c"], [0, 1, 0, 1]) == 0      # voice 3 (highest) holds "c": the node keeps "c"
        o1, _ = rt.render_voices(3, 1, x[:, :, :3 * 512])
        if prune:
            rt.prune_shared_resources()
            assert "b" not in rt.get_shared_resource_map_keys()
        o2, _ = rt.render_voices(nb - 3, 1, x[:, :, 3 * 512:])
        outs.append(np.concatenate([o1, o2], axis=2))
    assert np.array_equal(outs[0], outs[1])


def test_1024_voices_over_64_long_irs():
    n, k, nb = 1024, 64, 40
    res = {f"r{i}": np.asarray(graphs.lcg_ir(16384, seed=i + 1), dtype=np.float32) for i in range(k)}
    idx = np.random.default_rng(31).integers(0, k, size=n)
    rt, cid, batch = runtime(n, res, "r0")
    names = list(res)
    assert rt.set_path_per_voice(cid, names, idx) == 0
    assert convolvers(rt)[0]["irs"] == k and len(rt.describe()["groups"]) == 1
    x = noise(n, nb * 512, seed=37)
    got, _ = rt.render_voices(nb, 1, x)
    sample = np.random.default_rng(41).choice(n, size=16, replace=False)
    ref = reference(batch, cid, [names[idx[v]] for v in sample], {names[idx[v]]: res[names[idx[v]]] for v in sample} | {"r0": res["r0"]},
                    x[sample], nb)
    check(got[sample], ref)
