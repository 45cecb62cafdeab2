"""The column accounting of `modkit pileup` (observed codes, NoCall and diff counts, strand rules, motif rows, combined strands)
against an independent column-wise model (pileupmodel.py), on reads of depth above 1. This file holds the corpus the GPU suite
(test_gpu_pileup_columns.py) shares and the CPU checks: the model reproduces the reference's FeatureVector known answers and
every golden bedMethyl of its own test suite byte for byte, agrees with the oracle on the corpus under every flag set, and
the corpus reaches what it is meant to (the census)."""
import functools
import os
import random
import re
import subprocess

import pytest

import bamio
import pileupmodel as pm
from conftest import FIX, expand_args, golden_cases, run_oracle, same_text

# ---------------------------------------------------------------------------------------------------------------------------
# the model against the reference's own known answers and goldens


def fv_add(fv, aln, feature, read_strand, rule):
    fv.add_feature(aln, feature, read_strand, rule)


def test_feature_vector_known_answers():
    """test_feature_vector_basic and test_feature_vector_with_strand_rules (pileup/mod.rs:1038-1178)."""
    P, N, B = pm.POS, pm.NEG, pm.BOTH
    can, mod = lambda b: ("modcall", ("canonical", b), b), lambda c, b: ("modcall", ("mod", c), b)
    fv = pm.FeatureVector()
    for aln, feat in ((P, pm.nocall("A")), (P, can("C")), (P, mod("m", "C")), (P, mod("m", "C")), (P, pm.nocall("C")),
                      (N, pm.nocall("G")), (N, pm.nocall("G"))):
        fv_add(fv, aln, feat, P, B)
    rows = fv.decode({"C": {"m", "h"}}, {}, False, None, None)
    assert len(rows) == 2 and all(r.cov == 3 and r.n_nocall == 1 and r.n_diff == 1 and r.strand == P for r in rows)
    assert [r.code for r in rows] == ["h", "m"]
    fv = pm.FeatureVector()
    for aln, feat in ((P, can("C")), (N, mod("m", "C")), (N, pm.nocall("G")), (N, pm.nocall("G"))):
        fv_add(fv, aln, feat, P, B)
    rows = fv.decode({"C": {"m", "h"}}, {"C": {"m", "h"}}, False, None, None)
    assert len(rows) == 4 and all(r.n_diff == 2 for r in rows if r.strand == N)
    fv = pm.FeatureVector()
    fv_add(fv, P, mod("m", "C"), P, P)
    fv_add(fv, N, mod("m", "C"), P, P)                            # the wrong strand for a Positive rule: ignored
    rows = fv.decode({"C": {"m"}}, {}, False, None, None)
    assert len(rows) == 1 and rows[0].n_mod == 1


def golden_args(case, oracle_exe):
    """A golden case's flags; a sampled-threshold case gets the thresholds the oracle estimates for it."""
    args = expand_args(case["args"])
    if "--no-filtering" in args:
        return args
    p = subprocess.run([oracle_exe, "pileup", "-t", "4"] + args + [os.path.join(FIX, case["bam"]), os.devnull], capture_output=True, text=True)
    th = re.findall(r"Using filter threshold (\S+) for (\S+)\.", p.stderr)
    assert th, p.stderr
    return args + sum((["--filter-threshold", "%s:%s" % (b, t)] for t, b in th), [])


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["name"])
def test_model_matches_reference_golden(case, oracle_exe):
    got = pm.bedmethyl(os.path.join(FIX, case["bam"]), golden_args(case, oracle_exe))
    assert same_text(got, open(os.path.join(FIX, case["golden"])).read())


@pytest.fixture
def deletion_on_read_strand(monkeypatch):
    """A mistake put into the model: a deletion added with its read's strand instead of Positive."""
    orig = pm.FeatureVector.add_feature

    def add(self, aln, feature, read_strand, rule):
        orig(self, aln, feature, aln if feature == pm.DELETE else read_strand, rule)
    monkeypatch.setattr(pm.FeatureVector, "add_feature", add)


@pytest.fixture
def rows_only_for_called_codes(monkeypatch):
    """A mistake put into the model: a row only for the codes some read called at the position, not every observed code."""
    orig = pm.FeatureVector.add_tally_to_counts

    def add(out, tally, strand, observed, combine_mods, motif_idxs):
        called = {b: {s[1] for s in states if s[0] == "mod"} for b, states in tally.modcall_counts.items()}
        orig(out, tally, strand, {b: c & called.get(b, set()) for b, c in observed.items()}, combine_mods, motif_idxs)
    monkeypatch.setattr(pm.FeatureVector, "add_tally_to_counts", staticmethod(add))


def goldens_differing(oracle_exe):
    return [c["name"] for c in golden_cases() if pm.bedmethyl(os.path.join(FIX, c["bam"]), golden_args(c, oracle_exe)) !=
            open(os.path.join(FIX, c["golden"])).read()]


def test_model_with_deletion_on_read_strand_fails_goldens(deletion_on_read_strand, oracle_exe):
    """The model checks the deletion rule rather than mirroring the code: with the mistake, a golden disagrees."""
    assert goldens_differing(oracle_exe)


def test_model_with_rows_only_for_called_codes_fails_goldens(rows_only_for_called_codes, oracle_exe):
    assert goldens_differing(oracle_exe)


# ---------------------------------------------------------------------------------------------------------------------------
# the corpus

class Corpus:
    """Contigs and reads. Each read: (family, flag, MM text, record). Read names are unique (the read cache keys on the name)."""

    def __init__(self):
        self.contigs, self.reads, self.probes = {}, [], []

    def contig(self, name, seq):
        self.contigs[name] = seq
        return list(self.contigs).index(name)

    def add(self, family, tid, pos, flag, cigar, seq, mm, ml, aux=()):
        name = "r%d" % len(self.reads)
        rec = bamio.make_record(tid, pos, flag, cigar, seq, mm=mm, ml=ml, aux=aux, name=name)
        self.reads.append((family, flag, mm, rec))

    def write(self, d):
        bam, fa = os.path.join(d, "cols.bam"), os.path.join(d, "cols.fa")
        refs = [(n, len(s)) for n, s in self.contigs.items()]
        bamio.bam_of(refs, [r for *_, r in self.reads]).write(bam, index=True)
        bamio.write_fasta(fa, self.contigs)
        return bam, fa


def read_seq(ref, pos, cigar, rng, subs=None):
    """A stored SEQ that matches `ref` along `cigar` (inserted and clipped bases random); subs {query index: base}."""
    out, r = [], pos
    for op, n in cigar:
        if op in "M=X":
            out.append(ref[r:r + n])
            r += n
        elif op in "DN":
            r += n
        elif op in "IS":
            out.append("".join(rng.choice("ACGT") for _ in range(n)))
    s = list("".join(out))
    for k, b in (subs or {}).items():
        s[k] = b
    return "".join(s)


def calls_on(seq, rev, base, rng, every=1, skip=()):
    """[(read position, ML byte)] at every `every`-th `base` of the read (read orientation), minus read positions in skip."""
    read = bamio.revcomp(seq) if rev else seq
    return [(q, rng.randrange(256)) for k, q in enumerate(i for i, c in enumerate(read) if c == base) if k % every == 0 and q not in skip]


def n_codes(header):
    codes = header[2:].rstrip("?.")
    return 1 if codes.isdigit() else len(codes)


def mm_of(seq, rev, lists, rng):
    """MM text and ML of lists [(header, base of the read, options)] with a call at every such base (one byte per code). Lists
    of one (base, strand) table share the 256 so that their probabilities at a position sum to at most 1: the read is used."""
    share = {}
    for h, _, _ in lists:
        share[h[:2]] = share.get(h[:2], 0) + n_codes(h)

    def probs(h):
        v = tuple(rng.randrange(256 // share[h[:2]]) for _ in range(n_codes(h)))
        return v[0] if len(v) == 1 else v
    return bamio.mm_for(seq, rev, [(h, [(q, probs(h)) for q, _ in calls_on(seq, rev, b, rng, **o)]) for h, b, o in lists])

GEOMETRY_PAIRS = {(x, y, 0) for x in range(32) for y in range(x, 32)} | {(x, y, k) for x in range(32) for y in range(32) for k in (1, 2)}


@functools.lru_cache(maxsize=None)
def build_corpus():
    rng = random.Random(20261017)
    c = Corpus()
    # ---- family 1 and 3: scenes on homopolymer-C and CGCG stretches, one column P per scene --------------------------------
    scene = ("C" * 40 + "TTAATT" + "CGCGCGCGCG" + "AATT" + "A" * 20 + "TT") * 1
    n_scenes = 48
    scn = "".join(scene for _ in range(n_scenes)) + "T" * 50
    tid = c.contig("scn", scn)
    L = len(scene)

    def carrier(k, rev=False, lists=(("C+m?", "C", {}),)):
        s = k * L
        cig = [("M", L)]
        seq = read_seq(scn, s, cig, rng)
        mm, ml = mm_of(seq, rev, list(lists), rng)
        c.add("observed", tid, s, 16 if rev else 0, cig, seq, mm, ml)

    for k in range(n_scenes):
        s, P = k * L, k * L + 20
        kind = k % 24
        for rev in (False, True):
            carrier(k, rev)
        carrier(k, False, (("C+m?", "C", {}), ("A+a?", "A", {})))
        cig, subs, lists, flag = [("M", L)], {}, [("C+h?", "C", {"every": 3})], 0
        if kind == 0:                                            # a deletion at P
            cig = [("M", 20), ("D", 1), ("M", L - 21)]
        elif kind == 1:                                          # a mismatched base at P
            subs = {20: "A"}
        elif kind == 2:                                          # an N at P
            subs = {20: "N"}
        elif kind == 3:                                          # an IUPAC base at P
            subs = {20: "R"}
        elif kind == 4:                                          # a list that skips P
            lists = [("C+h?", "C", {"skip": (20,)})]
        elif kind == 5:                                          # an N op over P
            cig = [("M", 15), ("N", 10), ("M", L - 25)]
        elif kind == 6:                                          # a failed read: two lists over 1.01 at one position
            cig = [("M", L)]
            seq = read_seq(scn, s, cig, rng)
            mm = "C+h?,0;C+m?,0;"
            c.add("observed", tid, s, 0, cig, seq, mm, [250, 250])   # (failed on purpose)
            continue
        elif kind == 7:                                          # implicit without a mode flag (needs --force-allow-implicit)
            lists = [("C+h", "C", {"every": 4})]
        elif kind == 8:                                          # a reverse read
            flag = 16
        elif kind == 9:                                          # G-h on a forward read (the CGCG Gs)
            lists = [("C+m?", "C", {}), ("G-h?", "G", {})]
        elif kind == 10:                                         # implicit C+ and G- lists
            lists = [("C+h.", "C", {"every": 5}), ("G-h.", "G", {"every": 2})]
        elif kind == 11:                                         # implicit lists on a reverse read
            lists, flag = [("C+h.", "C", {"every": 5}), ("G-m.", "G", {"every": 2})], 16
        elif kind == 12:                                         # a list whose calls sit in the first 3 bases only (edge filter empties it)
            lists = [("C+h?", "C", {"skip": tuple(range(3, L))})]
        elif kind == 13:                                         # calls near the ends and inside: the edge filter drops some
            lists = [("C+h?", "C", {})]
        elif kind == 14:                                         # a ChEBI code next to letters
            lists = [("C+21839?", "C", {"every": 2}), ("C+m?", "C", {"every": 3})]
        elif kind == 15:                                         # duplex: C+m and G-m on one read
            lists = [("C+m?", "C", {}), ("G-m?", "G", {})]
        elif kind == 16:                                         # two codes, two primary bases, mismatching reads
            subs = {20: "A", 21: "A"}
            lists = [("C+m?", "C", {}), ("A+a?", "A", {})]
        elif kind == 17:                                         # a - list alone
            lists, flag = [("G-m?", "G", {})], 16
        elif kind == 18:                                         # three codes in one list
            lists = [("C+hmf?", "C", {"every": 2})]
        elif kind == 19:                                         # an aliased list pair
            lists = [("C+h?", "C", {}), ("C+m?", "C", {})]
        elif kind == 20:                                         # a + and a - list on one base: both call one position
            lists = [("C+m?", "C", {}), ("C-h?", "C", {})]
        elif kind == 21:
            lists, flag = [("C+m?", "C", {}), ("C-m?", "C", {"every": 2})], 16
        elif kind == 22:
            lists = [("G+h?", "G", {}), ("G-m?", "G", {})]
        else:
            cig, lists, flag = [("M", 20), ("D", 1), ("M", L - 21)], [("C-h?", "C", {}), ("C+m?", "C", {"every": 3})], 16
        seq = read_seq(scn, s, cig, rng, subs)
        rev = bool(flag & 16)
        mm, ml = mm_of(seq, rev, lists, rng)
        c.add("observed", tid, s, flag, cig, seq, mm, ml)
    # ---- family 3: one column at depth about 2 000, mixed states ---------------------------------------------------------------
    deep = "ACGTCCGGCCAT" * 4
    tid = c.contig("deep", deep + "T" * 20)
    for k in range(2000):
        rev = k % 3 == 0
        a = rng.randrange(0, 20)
        cig = [("M", 20), ("D", 2), ("M", 6)] if k % 7 == 0 else [("M", 28)]
        seq = read_seq(deep, a, cig, rng, {10: "A"} if k % 11 == 0 else None)
        lists = [("C+m?", "C", {}), ("C+h?", "C", {"every": 2})] if k % 5 else [("C+hm?", "C", {})]
        if k % 13 == 0:
            lists.append(("G-m?", "G", {}))
        mm, ml = mm_of(seq, rev, lists, rng)
        c.add("depth", tid, a, (16 if rev else 0) | (0x400 if k % 97 == 0 else 0), cig, seq, mm, ml)
    # ---- families 4-6: random sequence with motifs, reads of every list form, deletions, N ops, partition tags ---------------------
    mot = "".join(rng.choice("ACGT") for _ in range(30000))
    mot = mot[:5000] + "CGCGCGCG" * 20 + mot[5160:]
    tid = c.contig("mot", mot)
    forms = [[("C+m?", "C", {})], [("C+h?", "C", {}), ("C+m?", "C", {})], [("C+m?", "C", {}), ("A+a?", "A", {})],
             [("C+m.", "C", {"every": 2})], [("C+m?", "C", {}), ("G-m?", "G", {})], [("G-m?", "G", {})], [("C+m?", "C", {}), ("G-h.", "G", {"every": 3})],
             [("C+21839?", "C", {}), ("C+m?", "C", {"every": 2})], [("C+h?", "C", {"every": 2})],
             [("C+m?", "C", {}), ("C-m?", "C", {"every": 2})], [("G+h?", "G", {}), ("G-h?", "G", {})]]
    for k in range(2400):
        a = rng.randrange(0, len(mot) - 400)
        n = rng.randrange(60, 300)
        shape = k % 6
        if shape == 0:
            cig = [("M", n)]
        elif shape == 1:
            cig = [("S", 5), ("M", n // 2), ("D", 3), ("M", n // 2)]
        elif shape == 2:
            cig = [("M", n // 3), ("N", 40), ("M", n // 3)]
        elif shape == 3:
            cig = [("M", n // 2), ("I", 4), ("M", n // 2), ("S", 7)]
        elif shape == 4:
            cig = [("M", n // 4), ("D", 1), ("M", n // 4), ("D", 1), ("M", n // 4)]
        else:
            cig = [("M", n // 2), ("N", 7), ("M", n // 3)]
        rev = k % 2 == 1
        form = forms[k % len(forms)]
        seq = read_seq(mot, a, cig, rng, {rng.randrange(20, 50): "A"} if k % 17 == 0 else None)
        mm, ml = mm_of(seq, rev, form, rng)
        aux = (bamio.aux_i("HP", 1 + k % 2),) if k % 3 else ()
        c.add("motif", tid, a, 16 if rev else 0, cig, seq, mm, ml, aux)
    # ---- family 2: coverage runs (observed codes only) against the 32-position words ------------------------------------------
    # Every probe is the only reader of `h` over its stretch: a wrong bit in its coverage adds or drops an `h` row. A forward probe
    # calls `C+h` on its clipped first base, a reverse one `G-h` on its clipped last (stored) base, so `h` is observed over the
    # probe's aligned runs and called nowhere. A forward carrier over the same stretch calls `m` on every C, so every column has
    # a row. Probes are placed for the chunk origins of each setting in ORIGIN_SETS: two runs per probe, an N op between them.
    layout, cursor = [], 1
    for si, (name, (interval, chunk)) in enumerate(ORIGIN_SETS.items()):
        step = chunk // interval * interval
        need = sorted(GEOMETRY_PAIRS)
        rng.shuffle(need)

        def place(p, a, length):
            while True:
                cs = p // step * step
                if (p - cs) % 32 == a and p + length <= cs + step:
                    return p
                p += 1
        for t in range(0, len(need), 2):
            runs, p = [], cursor
            for a, b, k in need[t:t + 2]:
                length = b - a + 1 + 32 * k
                p = place(p, a, length)
                runs.append((p, p + length))
                p += length + 1
            layout.append((si, runs))
            cursor = runs[-1][1] + 2
    geo = "C" * (cursor + 50)
    tid = c.contig("geo", geo)
    for k, (si, runs) in enumerate(layout):
        a, e = runs[0][0], runs[-1][1]
        cig = [("M", e - a)]
        seq = read_seq(geo, a, cig, rng)
        mm, ml = mm_of(seq, False, [("C+m?", "C", {})], rng)
        c.add("geometry", tid, a, 0, cig, seq, mm, ml)
        rev = k % 2 == 1
        cig = [("M", runs[0][1] - runs[0][0])]
        for (x0, x1), (y0, y1) in zip(runs, runs[1:]):
            cig += [("N", y0 - x1), ("M", y1 - y0)]
        cig = cig + [("S", 1)] if rev else [("S", 1)] + cig
        seq = read_seq(geo, a, cig, rng)
        seq = seq[:-1] + "C" if rev else "C" + seq[1:]              # the clipped base: the read's first C (or G, reverse)
        c.probes.append((len(c.reads), tid, runs))
        mm = "G-h?,0;" if rev else "C+h.,0;" if k % 4 == 2 else "C+h?,0;"     # (implicit: canonical `h` calls at the other Cs)
        c.add("geometry", tid, a, 16 if rev else 0, cig, seq, mm, [200])
    return c


def chunk_origins(refs, interval, chunk_bp):
    """{tid: [chunk starts]}: consecutive intervals of one contig while their span stays within chunk_bp (the device pass's
    chunking, modkit_b200/csrc/host/pileup_run.hpp); bit k of a bitmap word is position origin + 32 w + k."""
    out = {}
    for tid, (_, ln) in enumerate(refs):
        starts, s = [], 0
        while s < ln:
            starts.append(s)
            e = s
            while e < ln and min(e + interval, ln) - s <= chunk_bp:
                e = min(e + interval, ln)
            s = max(e, min(s + interval, ln))
        out[tid] = starts
    return out


ORIGIN_SETS = {"default": (100000, 1 << 30), "i25_chunk990": (25, 990), "i88_chunk1000": (88, 1000)}


def geometry(runs, origins):
    """(first bit, last bit, class) of every run clipped to its chunk, class 0 inside one word, 1 across one word edge, 2 over a
    full word; the bits where the N ops between runs start and end; the count of probes that cross a chunk edge."""
    import bisect
    got, n_start, n_end, cuts = set(), set(), set(), 0
    for tid, rs in runs:
        st = origins[tid]
        rel = lambda p: (p - st[bisect.bisect_right(st, p) - 1]) & 31
        cuts += bisect.bisect_right(st, rs[0][0]) != bisect.bisect_right(st, rs[-1][1] - 1)
        for (_, x1), (y0, _) in zip(rs, rs[1:]):
            n_start.add(rel(x1))
            n_end.add(rel(y0 - 1))
        for a, b in rs:
            i = bisect.bisect_right(st, a) - 1
            while a < b:
                cs = st[i]
                ce = st[i + 1] if i + 1 < len(st) else 1 << 40
                y = min(b, ce)
                got.add(((a - cs) & 31, (y - 1 - cs) & 31, min(((y - 1 - cs) >> 5) - ((a - cs) >> 5), 2)))
                a, i = y, i + 1
    return got, n_start, n_end, cuts


def kernel_kind(mm):
    """The kernel paths a read takes: ("merged", one explicit list: one sorted run of calls that k_count_bases counts itself) or
    ("count_calls", several lists or an implicit one); ("fused", at most two codes per base, + strand, explicit, no N list)
    or ("list_mode", any other shape the fused kernel hands on)."""
    mm = mm.encode() if isinstance(mm, str) else mm
    lists = [p.split(b",")[0] for p in mm.split(b";") if p]
    implicit = any(not h.endswith(b"?") for h in lists)
    merged = "merged" if len(lists) == 1 and not implicit else "count_calls"
    bases = [h[:1] for h in lists]
    fused = all(h[1:2] == b"+" and h.endswith(b"?") and h[:1] != b"N" and len(h) <= 5 for h in lists) and len(set(bases)) == len(bases)
    return merged, "fused" if fused else "list_mode"


def test_corpus_census():
    c = build_corpus()
    kinds = {}
    for fam, flag, mm, _ in c.reads:
        for k in kernel_kind(mm) + ("reverse" if flag & 16 else "forward",):
            kinds.setdefault(fam, {}).setdefault(k, 0)
            kinds[fam][k] += 1
    print(kinds)
    for fam in ("observed", "depth", "motif", "geometry"):
        assert all(kinds[fam].get(k, 0) >= 20 for k in ("merged", "count_calls", "fused", "list_mode", "forward", "reverse")), (fam, kinds[fam])
    # the probes are live and each is the only reader of `h` over its stretch; the carriers carry `m` only
    opts = pm.Options(["--no-filtering"])
    refs, reads = bamio_records(c)
    live, spans = [], []
    for k, r in enumerate(reads):
        if r.tid != refs.index(("geo", len(c.contigs["geo"]))):
            continue
        st = pm.add_record(r, opts)
        codes = set().union(*st.codes[pm.POS].values(), *st.codes[pm.NEG].values())
        explicit_probe = codes == {"h"} and not r.mm.endswith(b".,0;")
        assert not st.skipped and codes in ({"m"}, {"h"}) and not (explicit_probe and any(st.calls[pm.POS].values()) or any(st.calls[pm.NEG].values())), (k, codes)
        if codes == {"h"}:
            live.append(k)
            spans.append((r.pos, r.end))
    assert sorted(live) == sorted(k for k, _, _ in c.probes)
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))      # no two probes share a column
    runs = [(tid, rs) for _, tid, rs in c.probes]
    for name, (interval, chunk) in ORIGIN_SETS.items():
        got, n_start, n_end, cuts = geometry(runs, chunk_origins(refs, interval, chunk))
        missing = GEOMETRY_PAIRS - got
        assert not missing, (name, len(missing), sorted(missing)[:8])
        assert len(n_start) == 32 and len(n_end) == 32, (name, len(n_start), len(n_end))
        assert name == "default" or cuts >= 100, (name, cuts)


def bamio_records(c):
    """(refs, raw records) of a corpus, for pileupmodel.load_bam."""
    return [(n, len(s)) for n, s in c.contigs.items()], [pm.Read(r) for *_, r in c.reads]


# ---------------------------------------------------------------------------------------------------------------------------
# the model against the oracle on the corpus

FLAG_SETS = [
    ("all", ["--no-filtering"]),
    ("all_force", ["--no-filtering", "--force-allow-implicit"]),
    ("edge", ["--no-filtering", "--force-allow-implicit", "--edge-filter", "3"]),
    ("ignore_h", ["--no-filtering", "--force-allow-implicit", "--ignore", "h"]),
    ("thresholds", ["--filter-threshold", "0.7", "--filter-threshold", "A:0.6", "--mod-thresholds", "m:0.8", "--force-allow-implicit"]),
    ("i25", ["--no-filtering", "--force-allow-implicit", "-i", "25"]),
    ("cpg", ["--no-filtering", "--force-allow-implicit", "--cpg", "--ref", "FA"]),
    ("cpg_i88", ["--no-filtering", "--cpg", "--ref", "FA", "-i", "88"]),
    ("motifs", ["--no-filtering", "--force-allow-implicit", "--motif", "CHH", "0", "--motif", "GATC", "1", "--motif", "RGY", "1", "--ref", "FA"]),
    ("cgcg", ["--no-filtering", "--force-allow-implicit", "--motif", "CG", "0", "--motif", "CGCG", "2", "--ref", "FA"]),
    ("include", ["--no-filtering", "--force-allow-implicit", "--include-bed", "BED"]),
    ("cpg_include", ["--no-filtering", "--force-allow-implicit", "--cpg", "--ref", "FA", "--include-bed", "BED"]),
    ("cpg_combine", ["--no-filtering", "--force-allow-implicit", "--cpg", "--combine-strands", "--ref", "FA"]),
    ("cpg_combine_i25", ["--no-filtering", "--force-allow-implicit", "--cpg", "--combine-strands", "--ref", "FA", "-i", "25"]),
    ("cgcg_combine", ["--no-filtering", "--force-allow-implicit", "--motif", "CG", "0", "--motif", "CGCG", "2", "--combine-strands", "--ref", "FA"]),
    ("combine_mods", ["--no-filtering", "--force-allow-implicit", "--combine-mods"]),
    ("combine_mods_strands", ["--no-filtering", "--force-allow-implicit", "--combine-mods", "--cpg", "--combine-strands", "--ref", "FA"]),
]


def write_bed(path):
    """+, -, . and BED3 intervals over the scenes and the motif contig."""
    lines = []
    for k, s in enumerate(range(0, 30000, 700)):
        strand = "+-.3"[k % 4]
        lines.append("mot\t%d\t%d" % (s, s + 300 + k) + ("" if strand == "3" else "\tx\t0\t%s" % strand))
    for k, s in enumerate(range(0, 3200, 160)):
        lines.append("scn\t%d\t%d\tx\t0\t%s" % (s + 15, s + 40, "+-."[k % 3]))
    lines.append("deep\t0\t48\tx\t0\t.")
    lines.append("geo\t100\t20000")
    open(path, "w").write("\n".join(lines) + "\n")


@pytest.fixture(scope="session")
def corpus_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("cols")
    c = build_corpus()
    bam, fa = c.write(str(d))
    bed = os.path.join(str(d), "inc.bed")
    write_bed(bed)
    return c, bam, fa, bed


def flags_of(name, fa, bed):
    return [fa if f == "FA" else bed if f == "BED" else f for f in dict(FLAG_SETS)[name]]


_MODEL = {}


def model_text(bam, flags):
    key = (bam, tuple(flags))
    if key not in _MODEL:
        _MODEL[key] = pm.bedmethyl(pm.load_bam(bam), flags)
    return _MODEL[key]


@pytest.mark.parametrize("name", [n for n, _ in FLAG_SETS])
def test_model_matches_oracle(name, corpus_files, oracle_exe, tmp_path):
    _, bam, fa, bed = corpus_files
    flags = flags_of(name, fa, bed)
    exp = run_oracle(oracle_exe, flags, bam, str(tmp_path / "o.bed"))
    assert exp.count("\n") > 100
    assert same_text(model_text(bam, flags), exp)


def test_model_matches_oracle_partitions(corpus_files, oracle_exe, tmp_path):
    """--partition-tag HP: reads of keys 1 and 2 share columns with each other and with untagged reads."""
    from conftest import read_dir
    _, bam, fa, bed = corpus_files
    flags = ["--no-filtering", "--force-allow-implicit", "--partition-tag", "HP"]
    p = subprocess.run([oracle_exe, "pileup", "-t", "4"] + flags + [bam, str(tmp_path / "part")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    exp = read_dir(str(tmp_path / "part"))
    assert sorted(exp) == ["1.bed", "2.bed", "ungrouped.bed"] and all(t.count("\n") > 1000 for t in exp.values())
    got = pm.partition_files(pm.load_bam(bam), flags)
    assert sorted(got) == sorted(exp)
    for name in exp:
        assert same_text(got[name], exp[name]), name


def test_corpus_reaches_plus_and_minus_calls_at_one_position():
    """Reads whose + and - lists on one base both call one position (the kernels' `nosub` case), forward and reverse."""
    c = build_corpus()
    opts = pm.Options(["--no-filtering", "--force-allow-implicit"])
    hits = {False: 0, True: 0}
    for r in bamio_records(c)[1]:
        st = pm.add_record(r, opts)
        if st.skipped:
            continue
        for base, calls in st.calls[pm.POS].items():
            if set(calls) & set(st.calls[pm.NEG].get(base, {})):
                hits[r.rev] += 1
    assert hits[False] >= 20 and hits[True] >= 20, hits
