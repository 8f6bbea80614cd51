"""CPU: the host side of voice resets (elem_b200_reset_voices) on plan-only engines — argument checks, what a reset must leave alone
(the voice groups, the programs, snapshot()), its launch count, and the render programs of every family, which the shadow rows of
`rand.seed` / `once.arm` must not change."""
import json
import os

import pytest

from elementary_b200 import Runtime, el, graphs
from elementary_b200.runtime import FLAG_MIX

HERE = os.path.dirname(os.path.abspath(__file__))


def plan(n_voices=45, **opts):
    return Runtime(48000.0, 512, n_voices, device=-1, plan_dry_run=1, **opts)


def synth(n_voices=45, **opts):
    rt = plan(n_voices, **opts)
    assert rt.apply_instructions(graphs.subsynth32()) == 0, rt.last_error()
    return rt


def state(rt):
    d = rt.describe()
    return d["groups"], rt.snapshot(0), rt.program_words(0).tolist()


def test_out_of_range_indices_change_nothing():
    rt = synth()
    before, launches = state(rt), rt.kernel_launches
    for bad in ([45], [-1], [0, 3, 45], [2**31 - 1], [-2**31], [2**40]):
        assert rt.reset_voices(bad) == -2, bad
    assert rt.kernel_launches == launches
    assert state(rt) == before


def test_empty_call_launches_nothing():
    rt = synth()
    launches = rt.kernel_launches
    assert rt.reset_voices([]) == 0
    assert rt.kernel_launches == launches


def test_unsorted_and_repeated_indices_are_accepted_and_cut_nothing():
    rt = synth(tile_width=4)
    rt.enqueue_block(0, 1, 512, flags=FLAG_MIX)
    before, launches = state(rt), rt.kernel_launches
    assert rt.reset_voices([44, 3, 3, 0, 17, 16, 44, 5]) == 0, rt.last_error()
    assert rt.kernel_launches == launches + 1        # one launch, whatever the number of voices and groups
    assert state(rt) == before                      # no group cut, nothing recompiled, same snapshot
    assert rt.reset_voices(list(range(45))) == 0
    assert rt.kernel_launches == launches + 2
    assert state(rt) == before


def test_one_launch_covers_every_group():
    rt = synth()
    assert rt.apply_instructions([[0, 0x7E000001, "sin"]], voices=(16, 45)) == 0, rt.last_error()   # cut: two groups
    assert rt.apply_instructions([[0, 0x7E000002, "sin"]], voices=(32, 45)) == 0, rt.last_error()   # three
    rt.enqueue_block(0, 1, 512, flags=FLAG_MIX)
    groups = rt.describe()["groups"]
    assert len(groups) == 3
    launches = rt.kernel_launches
    assert rt.reset_voices([40, 1, 20, 2]) == 0, rt.last_error()
    assert rt.kernel_launches == launches + 1
    assert rt.describe()["groups"] == groups


def test_reset_bytes_follow_the_plan():
    """A delay ring of `size` positions per lane, its write index, and nothing else: size * 4 + 4 bytes per voice."""
    rt = plan(8, tile_width=4)
    assert rt.apply_instructions(el.render(el.delay({"size": 100}, 10.0, 0.5, el.in_(0)))) == 0, rt.last_error()
    rt.enqueue_block(1, 1, 512, flags=FLAG_MIX)
    b0 = rt.reset_bytes_written
    assert rt.reset_voices([1, 6, 6]) == 0
    assert rt.reset_bytes_written - b0 == 2 * (100 * 4 + 4)


@pytest.mark.parametrize("kind", ["rand", "once"])
def test_shadow_props_are_checked_like_before(kind):
    """Setting the shadowed props keeps its return codes and per-voice behaviour (a value-only batch does not cut the group)."""
    rt = plan(8)
    node = el.rand(seed=3, key="r") if kind == "rand" else el.once({"arm": False}, el.in_(0))
    assert rt.apply_instructions(el.render(node)) == 0, rt.last_error()
    key, good, bad = ("seed", 7.0, "x") if kind == "rand" else ("arm", True, 1.0)
    assert rt.apply_instructions([[3, node.id(), key, good]], voices=(2, 5)) == 0
    assert len(rt.describe()["groups"]) == 1
    assert rt.apply_instructions([[3, node.id(), key, bad]]) == 5              # InvalidPropertyType
    if kind == "rand":
        assert rt.set_property_per_voice(node.id(), "seed", [1, 2, 3], 4) == 0


def test_program_words_unchanged_by_shadow_rows():
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_program_words import record
    want = json.load(open(os.path.join(HERE, "golden", "program_words.json")))
    got = record()
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k] == want[k], k
