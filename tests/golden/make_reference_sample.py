"""Generate tests/golden/reference_sample.npz: what the unmodified reference (oracle/_ref) produces in the `sample` node tests
(tests/sample_common.py), so that tests/test_sample_cpu.py also pins SampleModel where oracle/_ref cannot be built.  Stored per
scenario: the sha256 of each checked voice's float32 output 0 after the warm-up (truncated before its first read outside the buffer,
NaN after it), and the return codes of the prop cases.

Run where the reference sources are available to oracle/Makefile (REF=<path of the reference checkout>):
    python -c "import __graft_entry__ as g; g.build()"
    python tests/golden/make_reference_sample.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import oracle as orc                                  # noqa: E402
import sample_common                                              # noqa: E402
import test_sample_cpu                                            # noqa: E402


def compute():
    assert orc.ref_available(), "oracle/_ref/libelem_ref.so missing: build it where the reference sources are available"
    out = {}
    for sc in sample_common.scenarios() + [sample_common.many_voices()]:
        ref, _ = sc.reference(voices=test_sample_cpu.cpu_voices(sc))
        out["digest_" + sc.name] = np.array([sample_common.digest(r) for r in ref])
    out["prop_codes"] = np.array(json.dumps(test_sample_cpu.reference_prop_codes()))
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "reference_sample.npz"), **compute())
    print("wrote", os.path.join(HERE, "reference_sample.npz"))
