"""Functional graph front end that emits Elementary instruction batches.

Host-side mirror of the *output format* of the reference's JS front end (SURVEY.md Appendix B):
a batch is a JSON array of ``[0,id,type]`` create, ``[2,parent,child,chan]`` append,
``[3,id,key,value]`` set-property, ``[4,[roots]]`` activate, ``[5]`` commit, grouped in that order
(reference: js/packages/core/index.ts:43-49,122-130; Runtime.h:115-121).  The JS reconciler itself is out
of scope (SURVEY.md §2 row 16); this module exists so tests and benchmarks can *describe graphs the way the
reference's tests do* (``el.cycle(440)``, ``el.delay({size:10}, 0.5, 0, el.in_(channel=0))``) and feed the
resulting unchanged wire format to ``elementary_b200.Runtime`` and to the oracles.

Composite helpers follow the reference's definitions exactly, because the engine only ever sees native
nodes: ``cycle`` = sin(mul(2*pi, phasor(f)))  (js/packages/core/lib/oscillators.ts:39-41),
``saw`` = sub(mul(2, phasor(f)), 1) (:54-56), ``train`` = le(phasor(f), 0.5) (:27-29), etc.
"""
from __future__ import annotations

import json
import math
from typing import Any, Dict, Iterable, List, Optional, Sequence, Union

Number = Union[int, float]


class Node:
    """Immutable description of one graph node (type, props, ordered children)."""

    __slots__ = ("type", "props", "children", "_hash")

    def __init__(self, type_: str, props: Optional[Dict[str, Any]] = None, children: Sequence["Node"] = ()):
        self.type = type_
        self.props = dict(props or {})
        self.children = tuple(children)
        self._hash: Optional[int] = None

    # 31-bit structural id: equal sub-graphs share one node, like the reference's hashed NodeRepr
    # (src/HashUtils.res:8-44 uses FNV-1a too; the exact value is irrelevant to the engine, any int32 works).
    def id(self) -> int:
        if self._hash is None:
            h = 0x811C9DC5

            def mix(h: int, data: bytes) -> int:
                for b in data:
                    h ^= b
                    h = (h * 0x01000193) & 0xFFFFFFFF
                return h

            h = mix(h, self.type.encode())
            key = self.props.get("key")
            if key is not None:
                h = mix(h, b"k:" + str(key).encode())
            else:
                h = mix(h, json.dumps(self.props, sort_keys=True).encode())
            for c in self.children:
                h = mix(h, c.id().to_bytes(4, "little"))
            self._hash = h & 0x7FFFFFFF
        return self._hash

    def __repr__(self) -> str:  # pragma: no cover - debugging aid
        return f"Node({self.type}, {self.props}, n={len(self.children)})"


ElemNode = Union[Node, Number]


def resolve(x: ElemNode) -> Node:
    """Numbers become ``const`` nodes (js/packages/core/nodeUtils.ts resolve())."""
    if isinstance(x, Node):
        return x
    if isinstance(x, (int, float)):
        return Node("const", {"value": float(x)})
    raise TypeError(f"cannot resolve {x!r} to a graph node")


def create_node(type_: str, props: Optional[Dict[str, Any]], children: Iterable[ElemNode]) -> Node:
    return Node(type_, props or {}, [resolve(c) for c in children])


# --- native nodes -------------------------------------------------------------------------------------------
def const(value: Number, key: Optional[str] = None) -> Node:
    p: Dict[str, Any] = {"value": float(value)}
    if key is not None:
        p["key"] = key
    return Node("const", p)


def sr() -> Node:
    return Node("sr")


def in_(channel: int = 0, *children: ElemNode) -> Node:
    return create_node("in", {"channel": channel}, children)


def _unary(name):
    def f(x: ElemNode) -> Node:
        return create_node(name, {}, [x])
    f.__name__ = name
    return f


sin = _unary("sin"); cos = _unary("cos"); tan = _unary("tan"); tanh = _unary("tanh"); asinh = _unary("asinh")
ln = _unary("ln"); log = _unary("log"); log2 = _unary("log2"); ceil = _unary("ceil"); floor = _unary("floor")
round_ = _unary("round"); sqrt = _unary("sqrt"); exp = _unary("exp"); abs_ = _unary("abs")


def _binary(name):
    def f(a: ElemNode, b: ElemNode) -> Node:
        return create_node(name, {}, [a, b])
    f.__name__ = name
    return f


le = _binary("le"); leq = _binary("leq"); ge = _binary("ge"); geq = _binary("geq"); pow_ = _binary("pow")
eq = _binary("eq"); and_ = _binary("and"); or_ = _binary("or")


def _nary(name):
    def f(*args: ElemNode) -> Node:
        return create_node(name, {}, args)
    f.__name__ = name
    return f


add = _nary("add"); sub = _nary("sub"); mul = _nary("mul"); div = _nary("div"); mod = _nary("mod")
min_ = _nary("min"); max_ = _nary("max")


def phasor(rate: ElemNode) -> Node:
    return create_node("phasor", {}, [rate])


def syncphasor(rate: ElemNode, reset: ElemNode) -> Node:
    return create_node("sphasor", {}, [rate, reset])


def counter(gate: ElemNode) -> Node:
    return create_node("counter", {}, [gate])


def accum(x: ElemNode, reset: ElemNode) -> Node:
    return create_node("accum", {}, [x, reset])


def latch(t: ElemNode, x: ElemNode) -> Node:
    return create_node("latch", {}, [t, x])


def maxhold(props: Dict[str, Any], x: ElemNode, reset: ElemNode) -> Node:
    return create_node("maxhold", props, [x, reset])


def rand(seed: Optional[int] = None, key: Optional[str] = None) -> Node:
    p: Dict[str, Any] = {}
    if seed is not None:
        p["seed"] = seed
    if key is not None:
        p["key"] = key
    return Node("rand", p)


def pole(p: ElemNode, x: ElemNode) -> Node:
    return create_node("pole", {}, [p, x])


def env(atk: ElemNode, rel: ElemNode, x: ElemNode) -> Node:
    return create_node("env", {}, [atk, rel, x])


def z(x: ElemNode) -> Node:
    return create_node("z", {}, [x])


def delay(props: Dict[str, Any], length: ElemNode, fb: ElemNode, x: ElemNode) -> Node:
    return create_node("delay", props, [length, fb, x])


def sdelay(props: Dict[str, Any], x: ElemNode) -> Node:
    return create_node("sdelay", props, [x])


def prewarp(fc: ElemNode) -> Node:
    return create_node("prewarp", {}, [fc])


def mm1p(props: Dict[str, Any], fc: ElemNode, x: ElemNode) -> Node:
    return create_node("mm1p", props, [fc, x])


def svf(props: Dict[str, Any], fc: ElemNode, q: ElemNode, x: ElemNode) -> Node:
    return create_node("svf", props, [fc, q, x])


def svfshelf(props: Dict[str, Any], fc: ElemNode, q: ElemNode, gain_db: ElemNode, x: ElemNode) -> Node:
    return create_node("svfshelf", props, [fc, q, gain_db, x])


def biquad(b0: ElemNode, b1: ElemNode, b2: ElemNode, a1: ElemNode, a2: ElemNode, x: ElemNode) -> Node:
    return create_node("biquad", {}, [b0, b1, b2, a1, a2, x])


def tap_in(name: str) -> Node:
    return Node("tapIn", {"name": name})


def tap_out(name: str, x: ElemNode) -> Node:
    return create_node("tapOut", {"name": name}, [x])


def table(props: Dict[str, Any], t: ElemNode) -> Node:
    return create_node("table", props, [t])


def convolve(props: Dict[str, Any], x: ElemNode) -> Node:
    return create_node("convolve", props, [x])


def sample(props: Dict[str, Any], trigger: ElemNode, rate: Optional[ElemNode] = None) -> Node:
    """Sample playback (core.ts el.sample): plays the shared resource ``props["path"]`` from each rising edge of
    ``trigger``, at ``rate`` (1 without it).  Props: ``mode`` "trigger" / "gate" / "loop", ``startOffset``, ``stopOffset``."""
    return create_node("sample", props, [trigger] if rate is None else [trigger, rate])


def blepsaw(rate: ElemNode) -> Node:
    return create_node("blepsaw", {}, [rate])


def blepsquare(rate: ElemNode) -> Node:
    return create_node("blepsquare", {}, [rate])


def bleptriangle(rate: ElemNode) -> Node:
    return create_node("bleptriangle", {}, [rate])


# --- composites (reference: js/packages/core/lib/oscillators.ts, filters.ts, signals.ts) --------------------
def train(rate: ElemNode) -> Node:
    return le(phasor(rate), 0.5)


def cycle(rate: ElemNode) -> Node:
    return sin(mul(2.0 * math.pi, phasor(rate)))


def saw(rate: ElemNode) -> Node:
    return sub(mul(2, phasor(rate)), 1)


def square(rate: ElemNode) -> Node:
    return sub(mul(2, train(rate)), 1)


def triangle(rate: ElemNode) -> Node:
    return mul(2, sub(0.5, abs_(saw(rate))))


def noise(seed: Optional[int] = None) -> Node:
    return sub(mul(2, rand(seed)), 1)


def tau2pole(t: ElemNode) -> Node:
    # lib/filters.ts: exp(-1 / (t * sr))
    return exp(div(-1.0, mul(t, sr())))


def smooth(p: ElemNode, x: ElemNode) -> Node:
    # lib/filters.ts: pole(p, mul(sub(1, p), x))
    return pole(p, mul(sub(1, p), x))


# --- sequencing / control / analysis nodes (js/packages/core/lib/core.ts:17-66,103-153,304-355) ----------------
def time() -> Node:
    return Node("time", {})


def once(props: Dict[str, Any], x: ElemNode) -> Node:
    return create_node("once", props, [x])


def metro(props: Optional[Dict[str, Any]] = None) -> Node:
    return Node("metro", dict(props or {}))


def seq(props: Dict[str, Any], trigger: ElemNode, reset: ElemNode = 0) -> Node:
    return create_node("seq", props, [trigger, reset])


def seq2(props: Dict[str, Any], trigger: ElemNode, reset: ElemNode = 0) -> Node:
    return create_node("seq2", props, [trigger, reset])


def sparseq(props: Dict[str, Any], trigger: ElemNode, reset: ElemNode = 0) -> Node:
    return create_node("sparseq", props, [trigger, reset])


def sparseq2(props: Dict[str, Any], t: ElemNode) -> Node:
    return create_node("sparseq2", props, [t])


def meter(props: Dict[str, Any], x: ElemNode) -> Node:
    return create_node("meter", props, [x])


def snapshot(props: Dict[str, Any], trigger: ElemNode, x: ElemNode) -> Node:
    return create_node("snapshot", props, [trigger, x])


def scope(props: Dict[str, Any], *args: ElemNode) -> Node:
    return create_node("scope", props, list(args))


def capture(props: Dict[str, Any], g: ElemNode, x: ElemNode) -> Node:
    return create_node("capture", props, [g, x])


def fft(props: Dict[str, Any], x: ElemNode) -> Node:
    return create_node("fft", props, [x])


def select(g: ElemNode, a: ElemNode, b: ElemNode) -> Node:
    # lib/signals.ts: add(mul(g, a), mul(sub(1, g), b))
    return add(mul(g, a), mul(sub(1, g), b))


# --- renderer: Node graphs -> instruction batches -------------------------------------------------------------
class Renderer:
    """Minimal reconciler.  ``render(*roots)`` returns the instruction batch that brings the engine from the
    previously rendered graph to the new one: only unseen nodes are created, props are sent only when they
    changed, every call ends with ``[4,[roots]]`` and ``[5]`` (Reconciler.res:45-100, index.ts:122-130)."""

    def __init__(self, root_fade_in_ms: float = 20.0, root_fade_out_ms: float = 20.0):
        self._known: Dict[int, Dict[str, Any]] = {}
        self._fade_in = root_fade_in_ms
        self._fade_out = root_fade_out_ms

    def render(self, *graphs: ElemNode) -> List[list]:
        creates: List[list] = []
        appends: List[list] = []
        props: List[list] = []
        roots: List[int] = []
        visited: set = set()

        def visit(n: Node) -> None:
            nid = n.id()
            if nid in visited:
                return
            visited.add(nid)
            if nid not in self._known:
                creates.append([0, nid, n.type])
                self._known[nid] = {}
                for c in n.children:
                    appends.append([2, nid, c.id(), 0])
            known = self._known[nid]
            for k, v in n.props.items():
                if k == "key":
                    continue
                if k not in known or known[k] != v:
                    known[k] = v
                    props.append([3, nid, k, v])
            for c in n.children:
                visit(c)

        for i, g in enumerate(graphs):
            if g is None:
                continue
            root = Node("root", {"channel": i, "fadeInMs": self._fade_in, "fadeOutMs": self._fade_out}, [resolve(g)])
            visit(root)
            roots.append(root.id())

        return creates + appends + props + [[4, roots], [5]]


def render(*graphs: ElemNode) -> List[list]:
    """One-shot batch for a fresh engine."""
    return Renderer().render(*graphs)


def to_json(batch: List[list]) -> str:
    return json.dumps(batch)


def encode_binary(batch) -> bytes:
    """The instruction batch (list form, Appendix B of SURVEY.md) in the binary encoding of include/elem_b200.h ('EB2I' v1)."""
    import json as _json
    import struct
    out = [struct.pack("<III", 0x49324245, 1, len(batch))]
    for ins in batch:
        op = int(ins[0])
        out.append(struct.pack("<B", op))
        if op == 0:
            t = str(ins[2]).encode()
            out.append(struct.pack("<iH", int(ins[1]), len(t)) + t)
        elif op == 2:
            out.append(struct.pack("<iii", int(ins[1]), int(ins[2]), int(ins[3])))
        elif op == 3:
            k = str(ins[2]).encode()
            out.append(struct.pack("<iH", int(ins[1]), len(k)) + k)
            v = ins[3]
            if v is None:
                out.append(struct.pack("<B", 0))
            elif isinstance(v, bool):
                out.append(struct.pack("<BB", 1, 1 if v else 0))
            elif isinstance(v, (int, float)):
                out.append(struct.pack("<Bd", 2, float(v)))
            elif isinstance(v, str):
                b = v.encode()
                out.append(struct.pack("<BI", 3, len(b)) + b)
            elif isinstance(v, (list, tuple)) and all(isinstance(x, (int, float)) and not isinstance(x, bool) for x in v) and \
                    all(struct.unpack("<f", struct.pack("<f", float(x)))[0] == float(x) for x in v):
                out.append(struct.pack("<BI", 4, len(v)) + struct.pack("<%df" % len(v), *[float(x) for x in v]))
            else:
                b = _json.dumps(v).encode()
                out.append(struct.pack("<BI", 5, len(b)) + b)
        elif op == 4:
            ids = [int(x) for x in ins[1]]
            out.append(struct.pack("<I", len(ids)) + struct.pack("<%di" % len(ids), *ids))
        elif op == 5:
            pass
        else:
            raise ValueError(f"unknown opcode {op}")
    return b"".join(out)
