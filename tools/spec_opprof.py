#!/usr/bin/env python
"""Per-opcode cycle share of the SPECIALISED K1 on the flagship workload (bench.py: SUBSYNTH32, 48 kHz, 512-sample blocks, per-voice
f0) — the same clock64() brackets as tools/opprof.py, compiled into the NVRTC kernel by engine option spec_opprof (any library build).
Lane 0 of every warp adds each op's elapsed cycles to its opcode's counter; `loop` (slot 63) is the whole sample loop of a warp,
`prologue` (61) the staging of its state and parameter rows before the first tile, `writeback` (62) the state rows' way back to HBM.
Op shares are of the loop; the three parts are also given as shares of the warp's whole render (prologue + loop + write-back).
Usage: python tools/spec_opprof.py [voices=4096] [blocks=20]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from elementary_b200 import Runtime, graphs
from elementary_b200.runtime import FLAG_MIX

NAMES = ["END", "SEG", "FILL0", "COPY", "LOADIN", "CHAIN", "PHASOR", "SPHASOR", "COUNTER", "ACCUM", "LATCH", "MAXHOLD", "RAND", "POLE", "ENV", "BIQUAD",
         "PREWARP", "MM1P", "SVF", "SVFSHELF", "Z", "DELAY", "SDELAY", "TABLE", "BLEP", "TAPIN", "TAPOUT", "ROOT", "STOREBUF", "LOADBUF", "PROMOTE"]   # program.h
PROLOGUE, WRITEBACK, LOOP = 61, 62, 63

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
B = int(sys.argv[2]) if len(sys.argv) > 2 else 20
rt = Runtime(48000.0, 512, n, device=0, specialize=2, specialize_strict=1, spec_opprof=1)
assert rt.apply_instructions(graphs.subsynth32()) == 0
ida, idb = graphs.subsynth32_param_ids()
f0 = np.array([graphs.subsynth32_f0(v) for v in range(n)])
assert rt.set_property_per_voice(ida, "value", f0) == 0 and rt.set_property_per_voice(idb, "value", f0 * 1.007) == 0
for _ in range(4):
    rt.enqueue_block(0, 1, 512, FLAG_MIX)
rt.synchronize()
g = rt.describe()["groups"][0]
assert g.get("spec_state") == 2, g
rt.debug_opprof(True)
for _ in range(B):
    rt.enqueue_block(0, 1, 512, FLAG_MIX)
rt.synchronize()
p = rt.debug_opprof(True).astype(np.float64).reshape(64, 2)
ops, whole = p[:PROLOGUE, 0].sum(), p[LOOP, 0]
warps = max(1.0, p[LOOP, 1])
render = p[PROLOGUE, 0] + whole + p[WRITEBACK, 0]
print(json.dumps({"voices": n, "tile_width": g["tile_width"], "spec_regs": g.get("spec_regs"), "blocks": B,
                  "warp_cycles_per_block": whole / warps, "share_in_op_bodies": ops / max(1.0, whole),
                  "prologue_cycles_per_block": p[PROLOGUE, 0] / warps, "writeback_cycles_per_block": p[WRITEBACK, 0] / warps,
                  "prologue_share_of_render": p[PROLOGUE, 0] / max(1.0, render), "writeback_share_of_render": p[WRITEBACK, 0] / max(1.0, render)}))
rows = sorted(((p[op, 0], NAMES[op] if op < len(NAMES) else str(op), p[op, 1]) for op in range(PROLOGUE) if p[op, 1] > 0), reverse=True)
for c, name, cnt in rows:
    print(f"{name:9s} share {100 * c / whole:6.2f}% of the loop  cycles/warp-block {c / warps:9.0f}  dispatches/warp-block {cnt / warps:6.1f}")
print(f"{'rest':9s} share {100 * (whole - ops) / whole:6.2f}% of the loop  cycles/warp-block {(whole - ops) / warps:9.0f}  (outacc zeroing, epilogue, brackets)")
for slot, name in ((PROLOGUE, "prologue"), (LOOP, "loop"), (WRITEBACK, "writeback")):
    print(f"{name:9s} share {100 * p[slot, 0] / render:6.2f}% of the render  cycles/warp-block {p[slot, 0] / warps:9.0f}")
