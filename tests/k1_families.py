"""The K1 node families, shared by the K1 test matrix (tests/test_kernel_matrix_gpu.py) and the voice-group tests
(tests/test_voice_groups_gpu.py), the way tests/conv_exact.py serves K3.  Each family is one multi-root graph (<= 8 outputs) with its
keyed constants, seeds, resources, input generator and contract; next to them: the per-voice reference render, the GPU run helpers
and the checks of the contracts.

Contracts (DESIGN.md section 4, "Numerics"):

* ``exact``  -- np.array_equal against the reference for every voice and sample (NaN equals only NaN).  The kernels are compiled
  without FTZ, without fast math and without FMA contraction, and these nodes are sequences of IEEE float operations in the order
  of the reference: nothing may differ.  The interpreter and the specialised kernel must also be identical to each other.
* ``filter`` -- svf / svfshelf / mm1p compute in double.  The departures from the reference (Taylor tan, (pi fc) * (1 / sr) for
  pi fc / sr, rcp.approx + Newton, FMA contraction, the warp scan) are about 1e-16 relative (5e-13 for tan) of the double state.
  Three things amplify them: tan's condition number near Nyquist (fc at the sr / 2.0001 clamp: about 2e4), the resonance (q up
  to 20) and the cancellation of a highpass whose cutoff sits above the signal.  Measured on an H100, the worst case (highpass, fc
  at the clamp) is 1.7e-9 of the block peak, so: |gpu - ref| <= 1 ulp_f32(|ref|) + 1e-8 * block peak (DESIGN.md section 4).  The 1e-5 * block peak bound of the rest of the
  suite must also hold.
* ``math``   -- element-wise functions against a float64 NumPy evaluation of the same function on the same float32 inputs, within
  the maximum ulp error the CUDA 12 Math API documentation states for the single-precision function; results that are exact in
  IEEE arithmetic (sqrt, abs, floor, ceil, round, + - * /, fmod, min, max, compares) bit-exact against the reference.  A build with
  fast math (__sinf and friends) or FTZ (subnormal inputs and outputs flushed) breaks it.
* ``peak``   -- blep oscillators: |gpu - ref| <= 1e-5 * block peak, as in tests/test_parity_gpu.py.

The mix bus is compared with the float64 sum of the per-voice references in every run.
"""
import numpy as np

from elementary_b200 import Runtime, el
from helpers import block_peak_tolerance_check, oracle_cls

SR, BS = 48000.0, 512
N_VOICES = 45
CALLS = (512, 7, 100, 1, 333, 64, 63, 65, 8, 9, 255, 256, 257, 512)
FADE_END = 1024          # the 20 ms root fade-in (960 samples at 48 kHz) is over from here on: root out = node out * 1.0

GEOMETRIES = [(1, 0), (2, 0), (4, 0), (8, 0), (16, 0), (32, 0), (1, 4), (2, 8), (32, 4)]   # (tile_width, niter override)
DENSE_WIDTHS = (2, 4, 8, 16)
BUILDS = {
    "interp": {"specialize": 0},
    "spec": {"specialize": 2, "specialize_strict": 1, "specialize_max_words": 4096},
    "dense": {"specialize": 2, "specialize_strict": 1, "specialize_max_words": 4096, "spec_minblocks": 8},
}

IN0, IN1, IN2, IN3, IN4 = (el.in_(c) for c in range(5))


# ---- families ----------------------------------------------------------------------------------------------------------

class Family:
    def __init__(self, name, roots, n_in, contract, keyed=None, seeds=None, resources=None, inputs=None, math=None):
        self.name, self.roots, self.n_in, self.contract = name, roots, n_in, contract
        self.keyed = keyed or {}             # const key -> per-voice values (cycled)
        self.seeds = seeds or {}             # rand key -> function voice -> seed
        self.resources = resources or {}
        self.inputs = inputs or noise_inputs
        self.math = math                     # per root: ("exact",) or (float64 model, max ulp, input channels)
        self.batch = el.render(*roots)

    @property
    def n_out(self):
        return len(self.roots)

    def keyed_values(self, key, voices):
        vals = self.keyed[key]
        return [float(vals[v % len(vals)]) for v in voices]

    def voice_batch(self, v):
        b = [[3, el.const(0, key=k).id(), "value", self.keyed_values(k, [v])[0]] for k in self.keyed]
        b += [[3, el.rand(key=k).id(), "seed", float(f(v))] for k, f in self.seeds.items()]
        return b

    def setup(self, rt, v0=0, n=None):
        n = rt.num_voices - v0 if n is None else n
        voices = list(range(n))
        for k in self.keyed:
            assert rt.set_property_per_voice(el.const(0, key=k).id(), "value", self.keyed_values(k, voices), v0) == 0, rt.last_error()
        for k, f in self.seeds.items():
            assert rt.set_property_per_voice(el.rand(key=k).id(), "seed", [f(v) for v in voices], v0) == 0, rt.last_error()


def noise_inputs(fam, v, n):
    rng = np.random.default_rng(1000 + 7 * v)
    return rng.uniform(-1.0, 1.0, size=(fam.n_in, n)).astype(np.float32)


def math_inputs(fam, v, n):
    """Five channels of designed values, a quarter of them special, at random positions (so also after the fade-in):
    0 trig arguments (large ones included), 1 general (signed zeros, subnormals, +-0.5 / 1.5 / 2.5 for round, exp overflow),
    2 the log domain (zeros, negatives, subnormals), 3 pow bases / dividends, 4 exponents / divisors (integers and zero)."""
    rng = np.random.default_rng(5000 + 13 * v)
    specials = [
        [0.0, -0.0, 1e4, -1e4, 12345.678, 1e30, -1e30, 3.1415927, 1.5707964, -1.5707964, 1e-40, 1e-45, 100.5, 7e5],
        [0.0, -0.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.49999997, -0.49999997, 1e-40, -1e-40, 1e-45, 1.1754944e-38,
         88.0, 89.0, -104.0, -110.0, 1e30, 8388609.0],
        [0.0, -0.0, -1.0, 1.0, 1e-40, 1e-45, 1e30, 1.1754944e-38, 0.5, 3.4e38, 10.0, 1000.0],
        [0.0, -0.0, -2.0, -1.0, 1.0, 2.0, -0.5, -3.0, 1e-40, 2.5, -2.5],
        [0.0, -0.0, 0.5, -3.0, 3.0, 2.0, -2.0, 1.0, -1.0, 2.5, 6.0, -6.0],
    ]
    ranges = [(-10.0, 10.0), (-5.0, 5.0), (0.0, 100.0), (-4.0, 4.0), (-3.0, 3.0)]
    out = np.empty((fam.n_in, n), dtype=np.float32)
    for c in range(fam.n_in):
        x = rng.uniform(*ranges[c], size=n)
        if c == 4:                                           # integer exponents / divisors, zero among them
            ints = rng.integers(-6, 7, size=n).astype(np.float64)
            x = np.where(rng.random(n) < 0.5, ints, x)
        pick = rng.random(n) < 0.25
        x[pick] = rng.choice(np.array(specials[c]), size=int(pick.sum()))
        out[c] = x.astype(np.float32)
    return out


def impulse_inputs(fam, v, n):
    """channel 0: unit impulses after the fade-in (pole(0.5) decays through the subnormal range to zero within 150 samples);
    channel 1: values whose product with 1e-30 is subnormal."""
    rng = np.random.default_rng(9000 + v)
    out = np.zeros((2, n), dtype=np.float32)
    out[0, [FADE_END + 80 + v, 2000 + (v % 7)]] = 1.0
    out[1] = (rng.uniform(-1.0, 1.0, n) * 10.0 ** rng.uniform(-15.0, -4.0, n)).astype(np.float32)
    return out


def _pow_model(x, y):
    r = np.power(x, y)
    return np.where((x < 0) & (y != np.floor(y)), 0.0, r)


# CUDA 12 Math API documentation (CUDA C++ Programming Guide, "Mathematical Functions", single-precision table): maximum ulp
# error over the full range, without -use_fast_math.
ULP = {"sin": 2, "cos": 2, "tan": 4, "tanh": 2, "asinh": 3, "exp": 2, "ln": 1, "log": 2, "log2": 1, "pow": 4}
MODEL = {"sin": np.sin, "cos": np.cos, "tan": np.tan, "tanh": np.tanh, "asinh": np.arcsinh, "exp": np.exp, "ln": np.log,
         "log": np.log10, "log2": np.log2, "pow": _pow_model}
E = ("exact",)


def _t(name, *chans):
    return (MODEL[name], ULP[name], chans)


def _families():
    F = {}
    gate, gate2 = el.ge(IN1, -0.6), el.ge(IN2, 0.7)
    xq = el.round_(el.mul(8.0, IN0))                          # small integers: sums of delayed copies stay exact
    # PER - 1, PER, T - 1, T, T + 1 of every geometry (PER = 32 / L samples of a voice per slice, T samples per tile), a block
    sd_lengths = (1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 512)
    sd_sum = el.add(*[el.sdelay({"size": n}, xq) for n in sd_lengths])
    a, b = el.round_(el.mul(1.5, IN0)), el.round_(el.mul(1.5, IN1))
    cmp = el.add(el.le(a, b), el.mul(2.0, el.leq(a, b)), el.mul(4.0, el.ge(a, b)), el.mul(8.0, el.geq(a, b)),
                 el.mul(16.0, el.eq(a, b)), el.mul(32.0, el.and_(a, b)), el.mul(64.0, el.or_(a, b)))
    F["integer"] = Family("integer", [
        el.counter(gate),
        el.accum(IN0, gate2),
        el.latch(gate2, IN0),
        el.add(el.maxhold({}, IN0, gate2), el.mul(2.0, el.maxhold({"hold": 1.0}, IN0, 0.0))),
        el.add(el.once({"arm": True}, gate2), el.mul(2.0, el.z(IN0))),
        sd_sum,
        cmp,
        el.add(el.select(gate, IN0, IN1), el.mul(0.5, el.add(el.round_(el.mul(3.0, IN0)), el.floor(el.mul(3.0, IN1)),
                                                             el.ceil(el.mul(3.0, IN2)), el.abs_(IN0)))),
    ], 3, "exact")

    trig = el.train(el.const(2000.0, key="mx_tr"))
    rst = el.train(170.0)
    sp = [{"value": 1.0, "tickTime": 0}, {"value": 4.0, "tickTime": 3}, {"value": -2.0, "tickTime": 4}, {"value": 9.0, "tickTime": 11}]
    sp2 = [{"value": 0.5, "time": 0.002}, {"value": 2.0, "time": 0.004}, {"value": -1.0, "time": 0.011}, {"value": 3.0, "time": 0.02}]
    kf = [el.const(100.0, key=f"mx_f{i}") for i in range(5)]
    F["oscillators"] = Family("oscillators", [
        el.phasor(el.mul(2000.0, IN0)),                                   # audio-rate, negative frequencies
        el.phasor(kf[0]),
        el.add(el.phasor(kf[1]), el.phasor(kf[2]), el.phasor(kf[3]), el.phasor(kf[4])),   # a run of constant-frequency phasors
        el.syncphasor(kf[1], el.train(el.const(300.0, key="mx_sr"))),
        el.add(el.train(kf[2]), el.metro({"interval": 5.0})),
        el.time(),
        el.add(el.seq({"seq": [1.0, -2.0, 3.5, 0.25, 7.0], "hold": True, "loop": True}, trig, rst),
               el.mul(2.0, el.seq2({"seq": [0.5, 1.5, -2.5], "offset": 1}, trig, rst))),
        el.add(el.sparseq({"seq": sp, "loop": [1, 7]}, trig, 0.0), el.mul(4.0, el.sparseq2({"seq": sp2}, el.div(el.time(), el.sr())))),
    ], 1, "exact", keyed={
        "mx_f0": [-330.0, 0.0, 55.0, 440.0, 1234.5, 24000.0, 30000.0, 7.25],
        "mx_f1": [110.0, 220.5, -55.0, 1000.0, 3.0],
        "mx_f2": [333.3, 45.0, 12000.0, 0.5],
        "mx_f3": [77.0, 880.0, -1.0],
        "mx_f4": [2.0, 19999.0, 640.0, 41.0, 5.5, 6000.0],
        "mx_sr": [300.0, 37.0, 1200.0, 5.0],
        "mx_tr": [2000.0, 900.0, 4000.0, 150.0, 48000.0],
    })

    F["noise"] = Family("noise", [
        el.rand(seed=1, key="mx_r1"),
        el.sub(el.mul(2.0, el.rand(seed=2, key="mx_r2")), 1.0),
        el.mul(el.rand(seed=3, key="mx_r3"), IN0),
    ], 1, "exact", seeds={"mx_r1": lambda v: 1 + 7919 * v, "mx_r2": lambda v: 0x7FFF0000 - 104729 * v, "mx_r3": lambda v: v})

    kp = el.const(0.9, key="mx_p")
    F["recurrences"] = Family("recurrences", [
        el.pole(kp, IN0),
        el.env(el.const(0.9, key="mx_ea"), el.const(0.99, key="mx_er"), IN0),
        el.biquad(*[el.const(0.0, key=f"mx_b{i}") for i in range(5)], IN0),
        el.smooth(el.const(0.99, key="mx_sm"), IN0),
        el.pole(el.add(0.9, el.mul(0.09, IN1)), IN0),
        el.env(el.add(0.5, el.mul(0.45, IN1)), el.add(0.99, el.mul(0.0099, IN2)), IN0),
        el.biquad(el.mul(0.3, IN1), el.mul(0.2, IN2), 0.1, el.add(-0.5, el.mul(0.1, IN1)), el.add(0.25, el.mul(0.05, IN2)), IN0),
        el.smooth(el.add(0.95, el.mul(0.04, IN2)), IN0),
    ], 3, "exact", keyed={
        "mx_p": [0.0, 0.5, 0.9, 0.99, 0.999, -0.5, 1.0],
        "mx_ea": [0.1, 0.9, 0.99],
        "mx_er": [0.5, 0.999, 0.9999, 0.0],
        "mx_b0": [0.2, 1.0, 0.06, 0.5, 0.9], "mx_b1": [0.4, 0.0, 0.12, -1.0, -1.8], "mx_b2": [0.2, 0.0, 0.06, 0.5, 0.9],
        "mx_b3": [-0.5, 0.0, -1.6, -0.2, -1.78], "mx_b4": [0.3, 0.0, 0.8, 0.1, 0.81],
        "mx_sm": [0.9, 0.999, 0.5],
    })

    # per-voice delay times around the fast-path hazard window [hz + 1, size - hz - 1], hz = min(cnt, 32 / L), of every geometry:
    # consecutive voices (one warp) mix hazardous and safe read heads
    F["delay"] = Family("delay", [
        el.delay({"size": 64}, el.const(1.0, key="mx_d0"), el.const(0.3, key="mx_fb0"), IN0),
        el.delay({"size": 300}, el.add(150.0, el.mul(149.5, IN1)), 0.4, IN0),
        el.delay({"size": 64}, 0.0, 0.9, IN0),
        el.delay({"size": 1000}, el.const(100.0, key="mx_d1"), el.const(0.5, key="mx_fb1"), IN0),
        el.tap_out("mx_fb", el.add(IN0, el.mul(0.5, el.tap_in("mx_fb")))),
        el.delay({"size": 256}, el.const(200.0, key="mx_d2"), el.mul(0.9, IN1), IN0),
    ], 2, "exact", keyed={
        "mx_d0": [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 5.0, 8.0, 9.0, 16.0, 17.0, 17.5, 31.0, 32.0, 33.0, 47.0, 48.0, 55.0, 56.0,
                  59.0, 60.0, 61.0, 62.0, 62.5, 63.0, 64.0, 70.0, -3.0, 2.25, 30.75],
        "mx_fb0": [0.3, -0.7, 1.0, -1.0, 1.5, -2.0, 0.0],
        "mx_d1": [100.25, 511.5, 512.0, 513.0, 999.9, 33.3, 1000.0, 257.0],
        "mx_fb1": [0.5, -0.5, 0.99],
        "mx_d2": [200.0, 223.0, 224.0, 225.0, 238.0, 239.0, 240.0, 246.0, 247.0, 248.0, 250.0, 251.0, 252.0, 253.0, 254.0,
                  254.5, 255.0, 256.0, 1.0, 129.0, 127.5, 128.0],
    })

    def wave(n, k):
        return np.sin(np.linspace(0.0, 2.0 * np.pi * k, n, dtype=np.float64)).astype(np.float32) + np.float32(0.001 * k)

    pos0, pos1 = el.mul(1.2, IN0), el.add(0.5, el.mul(0.7, IN1))       # positions outside [0, 1] too
    F["table"] = Family("table", [
        el.table({"path": "mx_t8192"}, pos0),            # the program's first table: staged in shared memory (single-group launches)
        el.table({"path": "mx_t1000"}, pos1),
        el.table({"path": "mx_t3"}, pos0),
        el.table({"path": "mx_t1"}, pos1),
        el.table({"path": "mx_t8193"}, pos1),
    ], 2, "exact", resources={"mx_t8192": wave(8192, 3), "mx_t1000": wave(1000, 2), "mx_t3": np.array([1.0, -2.0, 3.0], np.float32),
                              "mx_t1": np.array([0.75], np.float32), "mx_t8193": wave(8193, 5)})

    fc, q = el.const(1000.0, key="mx_fc"), el.const(0.7, key="mx_q")
    modes = ["lowpass", "bandpass", "highpass", "notch", "allpass"]
    F["svf_keyed"] = Family("svf_keyed", [el.svf({"mode": m}, fc, q, IN0) for m in modes], 1, "filter", keyed={
        "mx_fc": [5.0, 20.0, 19.9, 100.0, 440.0, 1000.0, 5000.0, 12000.0, 23997.0, 23998.8, 30000.0, -50.0, 2500.0],
        "mx_q": [0.1, 0.25, 0.2499, 0.5, 0.7071, 1.0, 3.0, 10.0, 20.0, 20.01, 50.0],
    })
    fci, qi = el.mul(30000.0, IN1), el.add(10.0, el.mul(12.0, IN2))      # fc in [-30 k, 30 k], q in [-2, 22]: both clamps
    F["svf_inputs"] = Family("svf_inputs", [el.svf({"mode": m}, fci, qi, IN0) for m in modes], 3, "filter")

    sfc, sq, sg = el.const(900.0, key="mx_sfc"), el.const(0.8, key="mx_sq"), el.const(6.0, key="mx_sg")
    F["shelf_mm1p"] = Family("shelf_mm1p", [
        *[el.svfshelf({"mode": m}, sfc, sq, sg, IN0) for m in ("lowshelf", "highshelf", "bell")],
        *[el.mm1p({"mode": m}, el.prewarp(el.const(2000.0, key="mx_mfc")), IN0) for m in ("lowpass", "highpass", "allpass")],
        el.svfshelf({"mode": "bell"}, el.add(3000.0, el.mul(2900.0, IN1)), el.add(1.0, el.mul(0.9, IN2)), el.mul(18.0, IN1), IN0),
        el.mm1p({"mode": "lowpass"}, el.mul(1.2, IN2), IN0),                 # g beyond [0, 0.9999]
    ], 3, "filter", keyed={
        "mx_sfc": [10.0, 20.0, 900.0, 5000.0, 23998.8, 30000.0, 150.0],
        "mx_sq": [0.1, 0.25, 0.8, 5.0, 20.0, 40.0],
        "mx_sg": [-24.0, -6.0, 0.0, 3.0, 12.0, 24.0, -0.5, 9.0],
        "mx_mfc": [20.0, 200.0, 2000.0, 12000.0, 23000.0, 5.0],
    })

    # element-wise math: the CHAIN_REVERSED steps come from a fused operand in second position (sub / div / mod of x and f(y))
    F["math_a"] = Family("math_a", [el.sin(IN0), el.cos(IN0), el.tan(IN0), el.tanh(IN1), el.asinh(IN1), el.exp(IN1), el.ln(IN2),
                                    el.log(IN2)], 5, "math", inputs=math_inputs,
                         math=[_t("sin", 0), _t("cos", 0), _t("tan", 0), _t("tanh", 1), _t("asinh", 1), _t("exp", 1),
                               _t("ln", 2), _t("log", 2)])
    F["math_b"] = Family("math_b", [el.log2(IN2), el.pow_(IN3, IN4), el.sqrt(IN2), el.abs_(IN1), el.floor(IN1), el.ceil(IN1),
                                    el.round_(IN1), el.mod(IN3, IN4)], 5, "math", inputs=math_inputs,
                         math=[_t("log2", 2), _t("pow", 3, 4), E, E, E, E, E, E])
    F["math_c"] = Family("math_c", [el.add(IN1, IN3, IN4, 0.37), el.sub(IN1, el.floor(IN3)), el.sub(IN3, IN1, 0.25),
                                    el.mul(IN1, IN3, IN4), el.div(IN1, el.round_(IN4)), el.mod(IN1, el.floor(IN4)),
                                    el.min_(IN1, IN3, IN4), el.max_(IN1, IN3, IN4)], 5, "math", inputs=math_inputs, math=[E] * 8)
    ca, cb = el.round_(el.mul(2.0, IN3)), el.round_(el.mul(2.0, IN4))
    F["math_d"] = Family("math_d", [el.le(ca, cb), el.leq(ca, cb), el.ge(ca, cb), el.geq(ca, cb), el.eq(ca, cb), el.and_(ca, cb),
                                    el.or_(ca, cb), el.le(IN1, IN3)], 5, "math", inputs=math_inputs, math=[E] * 8)

    F["subnormal"] = Family("subnormal", [el.pole(0.5, IN0), el.mul(1e-30, IN1)], 2, "exact", inputs=impulse_inputs)

    F["analysis"] = Family("analysis", [
        el.meter({"name": "mx_m"}, el.mul(0.5, IN0)),
        el.snapshot({"name": "mx_s"}, el.train(el.const(500.0, key="mx_st")), IN0),
        el.scope({"name": "mx_sc", "channels": 2}, IN0, IN1),
        el.capture({"name": "mx_c"}, el.ge(IN1, 0.0), IN0),
        el.fft({"name": "mx_fft"}, IN1),
        el.in_(0, el.mul(0.25, IN1)),                     # an identity node with a child: copy
        el.create_node("pole", {}, [IN0]),                # a node without the inputs it needs: zeros
    ], 2, "exact", keyed={"mx_st": [500.0, 60.0, 3000.0]})

    bf = el.const(440.0, key="mx_bf")
    bfi = el.add(1500.0, el.mul(1400.0, IN0))
    F["blep"] = Family("blep", [el.blepsaw(bf), el.blepsquare(bf), el.bleptriangle(bf), el.blepsaw(bfi), el.blepsquare(bfi),
                                el.bleptriangle(bfi)], 1, "peak", keyed={"mx_bf": [55.0, 440.0, 1234.5, 5000.0, 12000.0]})
    return F


FAMILIES = _families()
MATH_FAMILIES = [f for f in FAMILIES if FAMILIES[f].contract == "math"]
RATE_FAMILIES = ["delay", "recurrences", "svf_keyed", "svf_inputs", "shelf_mm1p"]


# ---- reference (cached: it depends on neither geometry nor build) -----------------------------------------------------

_REF = {}


def family_inputs(fam, n_voices, n):
    if not fam.n_in:
        return None
    return np.stack([fam.inputs(fam, v, n) for v in range(n_voices)])


def reference(fam, calls=CALLS, sr=SR, bs=BS, n_voices=N_VOICES):
    """[voice, n_out, sum(calls)]: one reference instance per voice, fed the same process() lengths as the GPU."""
    key = (fam.name, sr, bs, tuple(calls), n_voices)
    if key not in _REF:
        total = sum(calls)
        inputs = family_inputs(fam, n_voices, total)
        outs = []
        for v in range(n_voices):
            o = oracle_cls()(sr, bs)
            for name, data in fam.resources.items():
                assert o.add_shared_resource(name, data)
            assert o.apply(fam.batch) == 0
            vb = fam.voice_batch(v)
            if vb:
                assert o.apply(vb) == 0
            parts, s = [], 0
            for n in calls:
                parts.append(o.process(None if inputs is None else inputs[v, :, s:s + n], fam.n_out, n))
                s += n
            outs.append(np.concatenate(parts, axis=1))
        _REF[key] = (np.stack(outs), inputs)
    return _REF[key]


# ---- GPU runs -----------------------------------------------------------------------------------------------------------

def make_runtime(fam, L, niter, build, sr=SR, bs=BS, n_voices=N_VOICES, **extra):
    opts = dict(BUILDS[build], tile_width=L, **extra)
    if niter:
        opts["niter"] = niter
    rt = Runtime(sr, bs, n_voices, device=0, **opts)
    for name, data in fam.resources.items():
        assert rt.add_shared_resource(name, data)
    assert rt.apply_instructions(fam.batch) == 0, rt.last_error()
    fam.setup(rt)
    rt.build = build
    assert rt.describe()["groups"][0]["tile_width"] == L       # a silently re-chosen geometry fails here
    return rt


def assert_build(rt):
    """After a block: the specialised arms really rendered with the specialised kernel (specialize=2 waits for it before the
    first block), not silently with the interpreter."""
    g = rt.describe()["groups"][0]
    if rt.build != "interp":
        assert g.get("spec_state") == 2, g


def run_calls(rt, fam, inputs, calls, n_out=None):
    n_out = n_out or fam.n_out
    vs, ms, s = [], [], 0
    for n in calls:
        v, m = rt.process_voices(None if inputs is None else inputs[:, :, s:s + n], n_out, n)
        vs.append(v)
        ms.append(m)
        s += n
    return np.concatenate(vs, axis=2), np.concatenate(ms, axis=1)


# ---- criteria -----------------------------------------------------------------------------------------------------------

def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def window_peak(ref, bs=BS):
    """max |ref| over each bs-sample window of the concatenated output (the last window may be shorter), per sample."""
    r = np.abs(np.asarray(ref, dtype=np.float64))
    n = r.shape[-1]
    out = np.empty_like(r)
    for s in range(0, n, bs):
        out[..., s:s + bs] = r[..., s:s + bs].max(axis=-1, keepdims=True)
    return out


def assert_exact(got, ref, what):
    if not np.array_equal(got, ref, equal_nan=True):
        bad = np.argwhere(~((got == ref) | (np.isnan(got) & np.isnan(ref))))
        v, c, t = bad[0]
        raise AssertionError(f"{what}: {len(bad)} samples differ; first voice {v} out {c} sample {t}: gpu {got[v, c, t]!r} "
                             f"ref {ref[v, c, t]!r}")


def check_filter(got, ref, what, bs=BS):
    g, r = got.astype(np.float64), ref.astype(np.float64)
    err = np.abs(g - r)
    bound = ulp32(r) + 1e-8 * window_peak(r, bs)
    worst_ulp = float((err / ulp32(r)).max())
    ratio = float((err / bound).max())
    v, c, t = np.unravel_index(int(np.argmax(err / bound)), err.shape)
    where = f"voice {v} out {c} sample {t}: gpu {got[v, c, t]!r} ref {ref[v, c, t]!r}, {int((err > bound).sum())} samples over"
    assert ratio <= 1.0, f"{what}: worst |gpu - ref| / (1 ulp + 1e-8 peak) = {ratio:.3g} (worst ulp {worst_ulp:.3g}) at {where}"
    tol = 1e-5 * window_peak(r, bs) + 1e-7
    assert (err <= tol).all(), f"{what}: worst err / (1e-5 peak) = {float((err / tol).max()):.3g} at {where}"
    return worst_ulp, ratio


def check_math(fam, got, ref, inputs, what):
    """Exact roots bit-exact against the reference everywhere; the others within their ulp bound of the float64 model after the
    fade-in (inputs are the float32 host inputs the kernel saw)."""
    worst = 0.0
    for c, spec in enumerate(fam.math):
        if spec[0] == "exact":
            assert_exact(got[:, c:c + 1], ref[:, c:c + 1], f"{what} root {c}")
            continue
        fn, max_ulp, chans = spec
        with np.errstate(all="ignore"):
            want = fn(*[inputs[:, ch, FADE_END:].astype(np.float64) for ch in chans])
        g = got[:, c, FADE_END:].astype(np.float64)
        w32 = want.astype(np.float32).astype(np.float64)
        fin = np.isfinite(w32)
        same_special = (g == w32) | (np.isnan(g) & np.isnan(w32))
        assert same_special[~fin].all(), f"{what} root {c}: non-finite results differ"
        err = np.abs(g[fin] - want[fin])
        u = err / ulp32(want[fin])
        bad = ~(u <= max_ulp)
        if bad.any():
            i = int(np.argmax(np.where(bad, u, -1.0)))
            args = [inputs[:, ch, FADE_END:][fin][i] for ch in chans]
            raise AssertionError(f"{what} root {c}: {int(bad.sum())} samples beyond {max_ulp} ulp, worst {u.max():.3g} ulp at "
                                 f"f{tuple(args)} = {want[fin][i]!r}, gpu {g[fin][i]!r}")
        worst = max(worst, float(u.max()) if u.size else 0.0)
    return worst


def check_mix(mix, ref, what):
    want = ref.astype(np.float64).sum(axis=0)
    scale = np.abs(ref).astype(np.float64).sum(axis=0)
    fin = scale < 1e38                     # no float32 partial sum can overflow (the math families render inf and NaN too)
    with np.errstate(invalid="ignore"):
        err = np.abs(mix.astype(np.float64) - want)[fin]
    assert (err <= 1e-6 * scale[fin] + 1e-7).all(), f"{what}: mix bus off by {err.max():.3g}"


def check_family(fam, got, mix, ref, inputs, what, bs=BS):
    """Applies the family's contract; returns (worst ulp or None, worst error / tolerance) for the report line."""
    if fam.contract == "exact":
        assert_exact(got, ref, what)
        stats = (0.0, 0.0)
    elif fam.contract == "filter":
        stats = check_filter(got, ref, what, bs)
    elif fam.contract == "math":
        stats = (check_math(fam, got, ref, inputs, what), 0.0)
    else:
        ok, worst, ex = block_peak_tolerance_check(got, ref, bs)
        assert ok, f"{what}: worst err/tol {worst:.3g}, bit-exact {ex:.4f}"
        stats = (None, worst)
    if mix is not None:
        check_mix(mix, ref, what)
    print(f"MATRIX {what}: worst_ulp={stats[0]} worst_err_over_tol={stats[1]:.3g}")
    return stats
