"""The specialised K1 against the interpreter, bit for bit, where the two sample-tile bodies of the specialised kernel and its two
root tails meet (render_kernel.cu, render_tile): a full tile (cnt == T) runs the program with cnt as a constant, a partial tile with
cnt at run time; a program with one root rendering one mix-only channel stores the tile's partial mix from OP_ROOT itself, every
other program and any block with per-voice outputs accumulates into outacc and runs the tile epilogue.  Block sizes that are not a
multiple of the tile length, and ragged process() calls, put partial tiles at every position of a block."""
import numpy as np
import pytest

from elementary_b200 import Runtime, el, graphs

SR = 48000.0
N_VOICES = 45            # odd: the last tile of every tile width has padding voices
RAGGED = (512, 7, 100, 1, 511)
BUILDS = {"interp": {"specialize": 0}, "spec": {"specialize": 2, "specialize_strict": 1, "specialize_max_words": 4096}}


def _k(v, key):
    return el.const(v, key=key)


def _filtered():
    """One root: a phasor through an svf and a one-pole, with per-voice parameters."""
    x = el.sub(el.mul(_k(2.0, "ft_two"), el.phasor(_k(110.0, "ft_f0"))), _k(1.0, "ft_one"))
    return el.pole(_k(0.3, "ft_p"), el.svf({"mode": "bandpass"}, _k(900.0, "ft_fc"), _k(2.0, "ft_q"), x))


def _second():
    return el.mul(_k(0.25, "sc_g"), el.delay({"size": 4800}, _k(700.5, "sc_len"), _k(0.3, "sc_fb"), el.phasor(_k(3.0, "sc_f"))))


PROGRAMS = {
    "subsynth32": (lambda: graphs.subsynth32(), 1),
    "filtered": (lambda: el.render(_filtered()), 1),
    "two_roots": (lambda: el.render(graphs.subsynth32_graph(), _second()), 2),
}


def _runtime(program, build, tile_width, block_size):
    batch, n_out = PROGRAMS[program]
    rt = Runtime(SR, block_size, N_VOICES, device=0, tile_width=tile_width, **BUILDS[build])
    assert rt.apply_instructions(batch()) == 0, rt.last_error()
    if program in ("subsynth32", "two_roots"):
        ida, idb = graphs.subsynth32_param_ids()
        f0 = np.array([graphs.subsynth32_f0(v) for v in range(N_VOICES)])
        assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
    else:
        v = np.arange(N_VOICES, dtype=np.float64)
        assert rt.set_property_per_voice(_k(0, "ft_f0").id(), "value", 55.0 * (1 + v % 13)) == 0
        assert rt.set_property_per_voice(_k(0, "ft_fc").id(), "value", 300.0 + 150.0 * v) == 0
    g = rt.describe()["groups"][0]
    assert g["tile_width"] == tile_width, g
    return rt, n_out


def _render(program, build, tile_width, block_size, calls, n_out=None, voices=False):
    rt, n = _runtime(program, build, tile_width, block_size)
    n_out = n_out or n
    vs, ms = [], []
    for c in calls:
        v, m = rt.process_voices(None, n_out, c, want_voices=voices)
        vs.append(v)
        ms.append(m)
    if build == "spec":
        assert rt.describe()["groups"][0].get("spec_state") == 2     # rendered by the specialised kernel, not the interpreter
    return (np.concatenate(vs, axis=2) if voices else None), np.concatenate(ms, axis=1)


def _same_bits(a, b, what):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    assert a.shape == b.shape, what
    diff = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
    assert diff.size == 0, f"{what}: {diff.size} samples differ, first at flat index {diff[0]}"


CASES = [
    # (block size, process() sizes): full tiles only, a partial last tile, a block longer than one launch's usual 512, ragged calls
    (512, (512,) * 3),
    (441, (441,) * 3),
    (1024, (1024, 1024)),
    (512, RAGGED),
    (1024, (1024, 7, 1000, 1, 1023)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width", [2, 32])
@pytest.mark.parametrize("program", ["subsynth32", "filtered"])
@pytest.mark.parametrize("block_size,calls", CASES, ids=[f"bs{b}-{'x'.join(map(str, c))}" for b, c in CASES])
def test_one_root_mix_only(program, tile_width, block_size, calls):
    """One root, one channel, mix only: the specialised kernel stores the partial mix from OP_ROOT."""
    _, want = _render(program, "interp", tile_width, block_size, calls)
    _, got = _render(program, "spec", tile_width, block_size, calls)
    _same_bits(got, want, f"{program} L={tile_width} bs={block_size} mix")


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width", [2, 32])
@pytest.mark.parametrize("block_size,calls", [(441, (441, 441)), (512, RAGGED)], ids=["bs441", "bs512-ragged"])
def test_old_tail_two_roots(tile_width, block_size, calls):
    """Two roots on two channels keep the accumulate-and-epilogue tail."""
    _, want = _render("two_roots", "interp", tile_width, block_size, calls)
    _, got = _render("two_roots", "spec", tile_width, block_size, calls)
    assert np.any(got[1] != 0.0)
    _same_bits(got, want, f"two roots L={tile_width} bs={block_size} mix")


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width", [2, 32])
@pytest.mark.parametrize("block_size,calls", [(441, (441, 441)), (1024, (1024, 7, 1000)), (512, RAGGED)], ids=["bs441", "bs1024", "bs512-ragged"])
def test_old_tail_per_voice_outputs(tile_width, block_size, calls):
    """Per-voice outputs requested: a one-root program keeps the old tail, voices and mix both bit for bit."""
    wv, wm = _render("subsynth32", "interp", tile_width, block_size, calls, voices=True)
    gv, gm = _render("subsynth32", "spec", tile_width, block_size, calls, voices=True)
    _same_bits(gv, wv, f"voices L={tile_width} bs={block_size}")
    _same_bits(gm, wm, f"mix L={tile_width} bs={block_size}")


@pytest.mark.gpu
@pytest.mark.parametrize("tile_width", [2, 32])
def test_old_tail_one_root_two_channels(tile_width):
    """One root but two output channels (the second silent): the old tail zero-fills the channel no root aims at."""
    _, want = _render("subsynth32", "interp", tile_width, 512, RAGGED, n_out=2)
    _, got = _render("subsynth32", "spec", tile_width, 512, RAGGED, n_out=2)
    assert not np.any(got[1])
    _same_bits(got, want, f"one root, two channels L={tile_width}")
