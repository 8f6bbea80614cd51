"""Per-voice sequences (Runtime.set_seq_per_voice) of seq, seq2, sparseq and sparseq2 on the GPU, bit for bit against a twin.

The twin is a runtime at tile width 1 whose voices got their sequences through JSON `seq` batches on voice sub-ranges (voice-group
cuts), the path the per-voice rows replace.  Its voices are permuted so that equal sequences are contiguous: it needs one group per
distinct sequence.  Both render the same per-voice trigger, reset and time inputs through process_voices calls of odd lengths, and
every voice must match its twin voice bit for bit (np.array_equal) — in every K1 tile geometry with the interpreter and in rotated
geometries with the specialised kernels, through live changes: a voice's sequence set again mid-run (the same one too), a whole-group
JSON `seq`, a sub-range JSON `seq` (a cut), a structural cut elsewhere, reset_voices and reset().  The pools hold empty sequences,
sequences of length 1, duplicated `time` / `tickTime` keys and unsorted input.  Where oracle/_ref is built, one geometry is also
checked against one reference instance per voice, at the exactness tests/control_common.py uses for the node.  Further cases: one-voice
graphs in the batched launch against the same graphs rendered alone, process_offline, the mix bus, and 4096 voices over 64 sequences.

ELEM_B200_SPECIALIZE=1 runs the interpreter arms on the specialised kernels as well."""
import numpy as np
import pytest

from elementary_b200 import Runtime, el
from k1_families import BUILDS, GEOMETRIES, assert_build, assert_exact, check_mix
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
SR, BS = 48000.0, 512
N_VOICES = 45
CALLS = (512, 7, 100, 1, 333, 512, 64, 257, 512, 255, 512, 512, 65, 512)
KINDS = ("seq", "seq2", "sparseq", "sparseq2")
EXACT = {"seq": True, "seq2": True, "sparseq": False, "sparseq2": False}   # tests/control_common.py: as its scenarios check the node

POOLS = {
    "seq": [[1.0, 2.0, 3.0, 4.0, 5.0], [], [7.0], [3.0, 1.0, 2.0], [1.0, 2.0, 3.0, 4.0, 5.0],
            [-1.0, -2.0, -3.0, -4.0, -5.0, -6.0, -7.0, -8.0, -9.0, -10.0], [0.5, 0.25]],
    "seq2": [[0.5, 1.5, -2.5], [], [9.0], [4.0, 4.0, 1.0, 3.0], [-0.125] * 3 + [8.0], [2.0, 3.0]],
    "sparseq": [[{"tickTime": 0, "value": 1.0}, {"tickTime": 3, "value": 2.0}, {"tickTime": 7, "value": -1.0}], [],
                [{"tickTime": 2, "value": 5.0}],
                [{"tickTime": 1, "value": 1.0}, {"tickTime": 1, "value": 9.0}, {"tickTime": 4, "value": 3.0}],
                [{"tickTime": 9, "value": 0.5}, {"tickTime": 0, "value": -4.0}, {"tickTime": 5, "value": 6.0}],
                [{"tickTime": 0, "value": 2.0}]],
    "sparseq2": [[{"time": 0.0, "value": 1.0}, {"time": 0.004, "value": 2.0}, {"time": 0.011, "value": -3.0}], [],
                 [{"time": 0.002, "value": 4.0}],
                 [{"time": 0.003, "value": 1.0}, {"time": 0.003, "value": 7.0}, {"time": 0.02, "value": -1.0}],
                 [{"time": 0.015, "value": 0.5}, {"time": 0.001, "value": -2.0}, {"time": 0.008, "value": 3.0}]],
}
INITIAL = {"seq": [10.0, 20.0, 30.0], "seq2": [0.75, -0.75], "sparseq": [{"tickTime": 1, "value": 8.0}],
           "sparseq2": [{"time": 0.006, "value": 6.0}]}


def graph(kind):
    """The node alone under a root; its inputs are host channels 0 (trigger, or time for sparseq2) and 1 (reset)."""
    if kind == "seq":
        node = el.seq({"seq": INITIAL[kind], "hold": True, "key": "n"}, el.in_(0), el.in_(1))
    elif kind == "seq2":
        node = el.seq2({"seq": INITIAL[kind], "hold": True, "key": "n"}, el.in_(0), el.in_(1))
    elif kind == "sparseq":
        node = el.sparseq({"seq": INITIAL[kind], "loop": [1, 6], "key": "n"}, el.in_(0), el.in_(1))
    else:
        node = el.sparseq2({"seq": INITIAL[kind], "interpolate": 1, "key": "n"}, el.in_(0))
    return node


def inputs(kind, n_voices, n):
    t = np.arange(n)[None, :]
    v = np.arange(n_voices)[:, None]
    x = np.zeros((n_voices, 2, n), dtype=np.float32)
    if kind == "sparseq2":
        x[:, 0] = (((t + 97 * v) % (1800 + 10 * v)) / SR).astype(np.float32)
    else:
        period = 40 + (v * 7) % 50
        x[:, 0] = (((t + 13 * v) % period) < period // 2).astype(np.float32)
        x[:, 1] = (((t + 101 * v) % 1500) < 3).astype(np.float32)
    return x


class Pair:
    """The runtime under test (`rt`, per-voice rows) and its twin (`tw`, tile width 1, sequences through JSON on voice sub-ranges);
    twin voice pos[v] renders voice v."""

    def __init__(self, kind, index, n_voices=N_VOICES, pool=None, **opts):
        self.kind, self.pool = kind, pool or POOLS[kind]
        node = graph(kind)
        self.nid, self.batch = node.id(), el.render(node)
        self.rt = Runtime(SR, BS, n_voices, device=0, **opts)
        assert self.rt.apply_instructions(self.batch) == 0, self.rt.last_error()
        index = np.asarray(index, dtype=np.int32)
        assert self.rt.set_seq_per_voice(self.nid, self.pool, index) == 0, self.rt.last_error()
        self.order = np.argsort(index, kind="stable")        # twin voice j renders voice order[j]
        self.pos = np.argsort(self.order)
        self.tw = Runtime(SR, BS, n_voices, device=0, tile_width=1)
        assert self.tw.apply_instructions(self.batch) == 0
        srt = index[self.order]
        starts = np.flatnonzero(np.r_[True, srt[1:] != srt[:-1]])
        for s, e in zip(starts, list(starts[1:]) + [n_voices]):
            assert self.tw.apply_instructions([[3, self.nid, "seq", self.pool[srt[s]]]], voices=(int(s), int(e))) == 0

    def per_voice(self, index, voice_begin):
        assert self.rt.set_seq_per_voice(self.nid, self.pool, index, voice_begin=voice_begin) == 0, self.rt.last_error()
        for i, k in enumerate(index):
            v = voice_begin + i
            p = int(self.pos[v])
            assert self.tw.apply_instructions([[3, self.nid, "seq", self.pool[k]]], voices=(p, p + 1)) == 0

    def json_seq(self, value, vb=0, ve=None):
        ve = self.rt.num_voices if ve is None else ve
        assert self.rt.apply_instructions([[3, self.nid, "seq", value]], voices=(vb, ve)) == 0, self.rt.last_error()
        for v in range(vb, ve):
            p = int(self.pos[v])
            assert self.tw.apply_instructions([[3, self.nid, "seq", value]], voices=(p, p + 1)) == 0

    def run(self, x, calls, script=None):
        """process_voices over `calls`; script[i](self) runs before call i.  Returns (got, twin [voice order], mix)."""
        got, twin, mix, s = [], [], [], 0
        for i, n in enumerate(calls):
            if script and i in script:
                script[i](self)
            g, m = self.rt.process_voices(x[:, :, s:s + n], 1, n)
            t, _ = self.tw.process_voices(x[self.order][:, :, s:s + n], 1, n)
            got.append(g)
            twin.append(t[self.pos])
            mix.append(m)
            s += n
        return np.concatenate(got, axis=2), np.concatenate(twin, axis=2), np.concatenate(mix, axis=1)


def live_script(L, n_voices=N_VOICES):
    a, b = (L, 3 * L) if 3 * L <= n_voices else (0, L)
    def set_again(p):                   # voices re-set mid-run, some to the sequence they already read
        p.per_voice([0, 0, 2, 1, 3], 2)
        p.per_voice([(v * 5) % len(p.pool) for v in range(7)], n_voices - 7)
    def whole_group(p):
        p.json_seq(p.pool[3])
        p.per_voice([1, 0, 4], 10)
    def sub_range(p):                   # a cut at tile boundaries; the voices outside keep their per-voice sequences
        p.json_seq(p.pool[0], a, b)
    c = b + L if b + L < n_voices else b
    def structural(p):                  # a node created on a voice range cuts a group elsewhere in the graph
        assert p.rt.apply_instructions([[0, 0x7E000001, "sin"]], voices=(c, n_voices)) == 0, p.rt.last_error()
        p.per_voice([2, 4], b - 1)
    def reset_voices(p):
        vs = [0, 5, 6, 17, n_voices - 1]
        assert p.rt.reset_voices(vs) == 0
        assert p.tw.reset_voices([int(p.pos[v]) for v in vs]) == 0
    def reset(p):
        p.rt.reset()
        p.tw.reset()
    return {2: set_again, 4: whole_group, 6: sub_range, 8: structural, 10: reset_voices, 12: reset}


def start_index(kind, n_voices):
    return [(v * 7 + v // 3) % len(POOLS[kind]) for v in range(n_voices)]


def _params():
    out = []
    for ki, kind in enumerate(KINDS):
        spec = [GEOMETRIES[(ki + 4 * j) % len(GEOMETRIES)] for j in range(2)]
        for L, niter in GEOMETRIES:
            out.append(pytest.param(kind, L, niter, "interp", id=f"{kind}-L{L}n{niter}-interp"))
            if (L, niter) in spec:
                out.append(pytest.param(kind, L, niter, "spec", id=f"{kind}-L{L}n{niter}-spec"))
    return out


@pytest.mark.parametrize("kind,tile_width,niter,build", _params())
def test_twin_bit_for_bit_with_live_changes(kind, tile_width, niter, build):
    opts = dict(BUILDS[build], tile_width=tile_width)
    if niter:
        opts["niter"] = niter
    p = Pair(kind, start_index(kind, N_VOICES), **opts)
    p.rt.build = build
    x = inputs(kind, N_VOICES, sum(CALLS))
    script = live_script(tile_width)
    script[1] = lambda p: assert_build(p.rt)   # the first call ran on the specialised kernel (groups recompiled later may not wait)
    got, twin, mix = p.run(x, CALLS, script)
    assert_exact(got, twin, f"{kind} L={tile_width} niter={niter} {build}")
    check_mix(mix, twin, f"{kind} mix")
    assert np.abs(got).max() > 0
    assert len(p.rt.describe()["groups"]) <= 4               # the sub-range batch and the structural one cut; per-voice calls do not


@pytest.mark.parametrize("kind", KINDS)
def test_against_the_reference(kind):
    """Where oracle/_ref is built: each voice against its own reference instance given the same sequences (no live changes)."""
    if not orc.ref_available():
        pytest.skip("the compiled reference is not built")
    n_voices = 12
    index = start_index(kind, n_voices)
    p = Pair(kind, index, n_voices=n_voices, tile_width=4)
    calls = CALLS[:8]
    x = inputs(kind, n_voices, sum(calls))
    got, twin, _ = p.run(x, calls)
    assert_exact(got, twin, f"{kind} twin")
    for v in range(n_voices):
        if not POOLS[kind][index[v]]:
            continue                    # the reference indexes an empty sequence (Core.h:497-500 and friends): not its domain
        o = orc.RefRuntime(SR, BS)
        assert o.apply(p.batch) == 0
        assert o.apply([[3, p.nid, "seq", POOLS[kind][index[v]]]]) == 0
        ref, s = [], 0
        for n in calls:
            ref.append(o.process(x[v, :, s:s + n], 1, n))
            s += n
        r = np.concatenate(ref, axis=1)
        if EXACT[kind]:
            assert np.array_equal(got[v], r), f"{kind} voice {v}: max diff {np.abs(got[v] - r).max()}"
        else:
            assert np.abs(got[v] - r).max() <= 1e-5 * max(np.abs(r).max(), 1e-30), f"{kind} voice {v}"


@pytest.mark.parametrize("kind", KINDS)
def test_process_offline(kind):
    p = Pair(kind, start_index(kind, N_VOICES), tile_width=8)
    n = 5 * BS + 100
    x = inputs(kind, N_VOICES, n)
    mix, voices = p.rt.process_offline(voice_inputs=x, num_outputs=1, want_voices=True)
    tmix, tv = p.tw.process_offline(voice_inputs=np.ascontiguousarray(x[p.order]), num_outputs=1, want_voices=True)
    assert_exact(voices, tv[p.pos], f"{kind} offline")
    check_mix(mix, tv, f"{kind} offline mix")


@pytest.mark.parametrize("stages", [0, 3])
def test_one_voice_graphs_in_the_batched_launch(stages):
    """One voice group per graph, launched together: each voice bit for bit what its graph renders alone."""
    n = 24
    kind_of = [KINDS[v % 4] for v in range(n)]
    rt = Runtime(SR, BS, n, device=0, pipeline_stages=stages)
    nodes = []
    for v in range(n):
        node = graph(kind_of[v])
        nodes.append(node.id())
        assert rt.apply_instructions(el.render(node), (v, v + 1)) == 0, rt.last_error()
        assert rt.set_seq_per_voice(node.id(), POOLS[kind_of[v]], [v % len(POOLS[kind_of[v]])], voice_begin=v) == 0
    assert len(rt.describe()["groups"]) == n
    x = np.stack([inputs(kind_of[v], n, sum(CALLS))[v] for v in range(n)])
    got, s = [], 0
    for c in CALLS:
        got.append(rt.process_voices(x[:, :, s:s + c], 1, c)[0])
        s += c
    got = np.concatenate(got, axis=2)
    for v in range(n):
        alone = Runtime(SR, BS, 1, device=0)
        assert alone.apply_instructions(el.render(graph(kind_of[v]))) == 0
        assert alone.set_seq_per_voice(nodes[v], POOLS[kind_of[v]], [v % len(POOLS[kind_of[v]])]) == 0
        want, s = [], 0
        for c in CALLS:
            want.append(alone.process_voices(x[v:v + 1, :, s:s + c], 1, c)[0])
            s += c
        assert_exact(got[v:v + 1], np.concatenate(want, axis=2), f"one-voice graph {v} ({kind_of[v]}) batched, stages={stages}")


@pytest.mark.parametrize("kind", KINDS)
def test_4096_voices_over_64_sequences(kind):
    n_voices = 4096
    rng = np.random.default_rng(7)
    base = POOLS[kind]
    pool = []
    for k in range(64):                # 64 distinct sequences from the pool, values scaled per k
        src = base[k % len(base)]
        if kind in ("seq", "seq2"):
            pool.append([float(np.float32(y * (1 + k))) for y in src])
        else:
            pool.append([dict(e, value=float(np.float32(e["value"] * (1 + k)))) for e in src])
    p = Pair(kind, rng.integers(0, 64, n_voices), n_voices=n_voices, pool=pool)
    assert len(p.rt.describe()["groups"]) == 1
    calls = (512, 100, 512, 412, 512)
    x = inputs(kind, n_voices, sum(calls))
    got, twin, mix = p.run(x, calls)
    assert_exact(got, twin, f"{kind} 4096 voices")
    check_mix(mix, twin, f"{kind} 4096 voices mix")
