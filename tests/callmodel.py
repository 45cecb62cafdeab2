"""An independent model of one base-modification call of `modkit pileup` (reference v0.4.4), in NumPy float32, written from
the reference's Rust sources:

    ML byte -> probability           quals_to_probs: (q + 0.5) / 256
    per-list tables                  get_base_mod_probs, BaseModProbs::new_init / add_base_mod_prob (mod_bam.rs:424-464)
    lists of one (strand, base)      combine_positions_to_probs, combine_checked, check (mod_bam.rs:629-656, 1037-1054)
    --ignore                         CollapseMethod::ReDistribute (mod_bam.rs:558-600)
    thresholded call                 MultipleThresholdModCaller::call (threshold_mod_caller.rs:28-63)
    arg-max call                     argmax_base_mod_call, canonical_prob (mod_bam.rs:489-509)

Every per-position map is an FxHashMap<ModCodeRepr, f32>: its iteration order, which sets both the order of the f32 sums and
who wins a tie, is that of hashbrown's table with rustc-hash 1.1's FxHasher (bucket = hash & mask, linear probe, iteration by
ascending bucket; 4 buckets for up to 3 codes, 8 from the 4th). Rust's `max` / `max_by` return the LAST of equal maxima, and
the canonical candidate is pushed after the mod codes, so it wins a tie with any of them.

Every arithmetic step is one explicit np.float32 operation. Beside it, `exact=True` runs the same steps on fractions.Fraction
(the f32 constants 1.01 and the thresholds taken at their f32 values): a call whose f32 answer differs from the exact one is
f32-decisive."""
from fractions import Fraction

import numpy as np

F32 = np.float32
MAX_PROB = F32(1.01)
K = 0x517cc1b727220a95
M64 = (1 << 64) - 1


def fx_hash(code):
    """FxHasher of a ModCodeRepr: the derived Hash writes the variant index (Code 0, ChEbi 1) as usize, then the char / u32."""
    h = 0
    for word in ((0, ord(code)) if isinstance(code, str) else (1, code)):
        h = ((((h << 5) | (h >> 59)) & M64) ^ word) * K & M64
    return h


def code_of(text):
    """ModCodeRepr of an MM / CLI code: one letter, or a ChEBI number (int)."""
    return int(text) if text.isdigit() else text


class FxMap:
    """The part of hashbrown's RawTable the reads reach: insertion with growth, lookup, iteration in bucket order."""

    def __init__(self, reserve=0):
        self.slots = [None] * (0 if reserve <= 0 else 4 if reserve < 4 else 8)
        self.vals = {}

    def _place(self, code):
        n = len(self.slots)
        s = fx_hash(code) & (n - 1)
        while self.slots[s] is not None:
            s = (s + 1) & (n - 1)
        self.slots[s] = code

    def insert(self, code, v):
        if code not in self.vals:
            cap = 0 if not self.slots else len(self.slots) - 1 if len(self.slots) < 8 else len(self.slots) // 8 * 7
            if len(self.vals) + 1 > cap:
                old = [c for c in self.slots if c is not None] if self.slots else []
                want = len(self.vals) + 1
                self.slots = [None] * (4 if want < 4 else 8 if want < 8 else 1 << (want * 8 // 7 - 1).bit_length())
                for c in old:
                    self._place(c)
            self._place(code)
        self.vals[code] = v

    def get(self, code):
        return self.vals.get(code)

    def items(self):
        return [(c, self.vals[c]) for c in self.slots if c is not None]

    def __len__(self):
        return len(self.vals)


class Arith:
    """float32 or exact arithmetic: one operation per call, nothing fused."""

    def __init__(self, exact):
        self.exact = exact

    def num(self, x):
        return Fraction(float(F32(x))) if self.exact else F32(x)

    def prob(self, q):
        return Fraction(2 * q + 1, 512) if self.exact else F32(F32(F32(q) + F32(0.5)) / F32(256.0))

    def add(self, a, b):
        return a + b if self.exact else F32(F32(a) + F32(b))

    def sub(self, a, b):
        return a - b if self.exact else F32(F32(a) - F32(b))

    def div(self, a, b):
        return a / b if self.exact else F32(F32(a) / F32(b))

    def sum(self, xs):
        s = self.num(0.0)
        for x in xs:
            s = self.add(s, x)
        return s


class ReadError(Exception):
    """The read fails as a whole (ProbaGreaterThanOne): none of its calls count."""


def position_maps(lists, ar):
    """{position: FxMap} of one (strand, base) table from [(codes, {position: (ML byte per code)})] in MM order.
    Raises ReadError when a repeated code or a combined position sums above 1.01."""
    agg = {}
    for codes, calls in lists:
        table = {}
        for pos in sorted(calls):
            for code, q in zip(codes, calls[pos]):
                p = ar.prob(q)
                m = table.get(pos)
                if m is None:                                   # BaseModProbs::new_init: FxHashMap::from_iter([(code, p)])
                    m = table[pos] = FxMap(reserve=1)
                    m.insert(code, p)
                else:                                           # add_base_mod_prob: only a repeated code is checked
                    cur = m.get(code)
                    cur = ar.num(0.0) if cur is None else cur
                    if ar.add(cur, p) > ar.num(MAX_PROB):
                        raise ReadError
                    m.insert(code, ar.add(cur, p))
        for pos, m in table.items():                            # combine_positions_to_probs
            a = agg.get(pos)
            if a is None:
                agg[pos] = m
                continue
            for code, p in m.items():                           # combine_checked
                cur = a.get(code)
                a.insert(code, ar.add(ar.num(0.0) if cur is None else cur, p))
            if ar.sum(v for _, v in a.items()) > ar.num(MAX_PROB):
                raise ReadError
    return agg


def redistribute(m, drop, ar):
    """CollapseMethod::ReDistribute(drop): the dropped code's probability shared by the other codes and the canonical base."""
    marginal = ar.sum(p for c, p in m.items() if c == drop)
    others = [(c, p) for c, p in m.items() if c != drop]
    share = ar.div(marginal, ar.add(ar.num(len(others)), ar.num(1.0)))
    out = FxMap()
    for c, p in others:
        out.insert(c, ar.add(p, share))
    return out


def canonical_prob(m, ar):
    return ar.sub(ar.num(1.0), ar.sum(p for _, p in m.items()))


class Caller:
    """MultipleThresholdModCaller: per-mod thresholds (a base letter is the any-mod code of that base), per-base thresholds,
    the default; Caller() is the pass-through of --no-filtering."""

    def __init__(self, per_mod=None, per_base=None, default=0.0):
        self.per_mod = {code_of(k): F32(v) for k, v in (per_mod or {}).items()}
        self.per_base = {k: F32(v) for k, v in (per_base or {}).items()}
        self.default = F32(default)

    def mod_threshold(self, code, base):
        for t in (self.per_mod.get(code), self.per_mod.get(base), self.per_base.get(base)):
            if t is not None:
                return t
        return self.default


def call(m, caller, base, ar):
    """('mod', code, p) / ('canonical', None, p) / ('fail', None, None) of one position map."""
    best = None
    for c, p in m.items():
        if p >= ar.num(caller.mod_threshold(c, base)):
            if best is None or p >= best[2]:                    # Iterator::max: the last of equal maxima
                best = ("mod", c, p)
    cp = canonical_prob(m, ar)
    if cp >= ar.num(caller.per_base.get(base, caller.default)):
        if best is None or cp >= best[2]:
            best = ("canonical", None, cp)
    return best or ("fail", None, None)


def argmax(m, ar):
    """(kind, code, value) of argmax_base_mod_call: the last maximal mod code if it beats the canonical probability."""
    cp = canonical_prob(m, ar)
    best = None
    for c, p in m.items():
        if best is None or p >= best[1]:                        # max_by: the last of equal maxima
            best = (c, p)
    if best is not None and best[1] > cp:
        return ("mod", best[0], best[1])
    return ("canonical", None, cp)


def read_calls(lists, caller, ignore=None, base="C", exact=False):
    """{position: (call, argmax, codes)} of one read's (strand, base) table (codes: the position's codes after the collapse), or
    None when the read fails as a whole."""
    ar = Arith(exact)
    try:
        maps = position_maps([([code_of(c) for c in codes], calls) for codes, calls in lists], ar)
    except ReadError:
        return None
    out = {}
    for pos, m in maps.items():
        if ignore is not None:
            m = redistribute(m, code_of(ignore), ar)
        out[pos] = (call(m, caller, base, ar), argmax(m, ar), frozenset(c for c, _ in m.items()))
    return out


def map_order(codes):
    """Iteration order of a map built by inserting `codes` in this order."""
    m = FxMap()
    for c in codes:
        m.insert(code_of(c) if isinstance(c, str) else c, 0)
    return [c for c, _ in m.items()]


def percentile(values, q):
    """percentile_linear_interp (thresholds.rs:17-39) over the sorted f32 values."""
    xs = sorted(F32(v) for v in values)
    q = F32(q)
    if len(xs) < 2:
        raise ValueError("not enough datapoints")
    if q == F32(1.0):
        return xs[-1]
    lq = F32(F32(len(xs) - 1) * q)
    g = F32(lq - F32(np.trunc(lq)))
    y0, y1 = xs[int(np.floor(lq))], xs[int(np.ceil(lq))]
    return F32(F32(y0 * F32(F32(1.0) - g)) + F32(y1 * g))
