"""Records tests/golden/program_words.json: the render program of every K1 node family (tests/k1_families.py) and of SUBSYNTH32 at
three tile widths, with the device-pointer words of the op headers masked.  It was recorded before voice resets added the shadow
rows of `rand.seed` and `once.arm` (rows outside every node's state rows), and tests/test_voice_reset_cpu.py checks that the
programs are still word for word the same.

    python tests/golden/make_program_words.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))                       # tests/: k1_families, helpers
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))      # the repository: elementary_b200

WIDTHS = (1, 4, 32)


def masked(words):
    """The program words up to and including the first OP_END, with each op header's device pointer (w4, w5) zeroed."""
    w = [int(x) for x in words]
    pc = 0
    while pc + 8 <= len(w):
        n = 8 + ((w[pc] >> 8) & 0xFF)
        w[pc + 4] = w[pc + 5] = 0
        if (w[pc] & 0xFF) == 0:
            break
        pc += n
    return w[:pc + 8]


def graphs_to_record():
    from elementary_b200 import graphs
    from k1_families import FAMILIES
    out = {name: (fam.batch, fam.resources) for name, fam in FAMILIES.items()}
    out["subsynth32"] = (graphs.subsynth32(), {})
    return out


def program(batch, resources, L):
    from elementary_b200 import Runtime
    rt = Runtime(48000.0, 512, 8, device=-1, tile_width=L)
    for name, data in resources.items():
        assert rt.add_shared_resource(name, data)
    assert rt.apply_instructions(batch) == 0, rt.last_error()
    return masked(rt.program_words(0))


def record():
    return {f"{name}/L{L}": program(batch, res, L) for name, (batch, res) in graphs_to_record().items() for L in WIDTHS}


if __name__ == "__main__":
    with open(os.path.join(HERE, "program_words.json"), "w") as f:
        json.dump(record(), f, separators=(",", ":"), sort_keys=True)
