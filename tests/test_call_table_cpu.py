"""The per-call probability arithmetic (ML byte -> probability, per-list sums and the 1.01 checks, ReDistribute, hash-map
iteration order, the thresholded and arg-max calls) on a call table: reads built so that every bedMethyl row holds exactly
one call, whose ML bytes walk the edges where that arithmetic goes wrong - every two-code pair up to a sum of 262, sums
that make a read fail, repeated codes, three and four codes on C with exact ties and f32 rounding, thresholds on the
1/1024 grid. This file holds the builder the GPU suite (test_gpu_call_table.py) shares and the CPU checks: the independent
model (callmodel.py) agrees with the oracle on every flag set, and the table reaches every family it is meant to."""
import functools
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

import callmodel as cm
from conftest import run_oracle
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)
from test_read_shapes_cpu import Genome

UNIT = "ACGA"        # one CpG per slot: the forward read's C, the reverse read's C (the reference G); no CpG across units
GAP = "TT"
CHEBI = "76792"      # a ChEBI code: bucket 2 of a 4-bucket table (f's), and of an 8-bucket one, where f moves to 6


def f32_text(x):
    """Shortest text that parses back to the same f32."""
    return np.format_float_positional(np.float32(x), unique=True, trim="-")


class Read:
    """One read of the table: `lists` = [(header, {slot: ML bytes of the header's codes})] in read orientation."""

    def __init__(self, family, lists, n_slots, rev):
        self.family, self.lists, self.n, self.rev = family, lists, n_slots, rev
        self.start = None

    def model_lists(self):
        """[(codes, {slot: bytes})] of the read's C+ lists for callmodel."""
        out = []
        for header, calls in self.lists:
            if header.startswith("C+"):
                body = header[2:-1]
                out.append(([body] if body.isdigit() else list(body), calls))
        return out

    def position(self, slot):
        """(reference position, strand) of the call at a slot."""
        if not self.rev:
            return self.start + 4 * slot + 1, "+"
        return self.start + 4 * (self.n - 1 - slot) + 2, "-"


class Table:
    def __init__(self, reads, thresholds):
        self.reads, self.thresholds = reads, thresholds


def two_code_reads(rng, reads, shape, pairs, per_read=48):
    """Grid pairs (a, b) as h, m bytes; shapes: sep (C+h? and C+m? at the same slots), comb (one C+hm? list), shift (sep,
    plus slots with only one of the two lists between the pairs)."""
    for k in range(0, len(pairs), per_read):
        chunk = pairs[k:k + per_read]
        if shape == "comb":
            lists = [("C+hm?", {i: ab for i, ab in enumerate(chunk)})]
            n = len(chunk)
        elif shape == "sep":
            lists = [("C+h?", {i: (a,) for i, (a, b) in enumerate(chunk)}), ("C+m?", {i: (b,) for i, (a, b) in enumerate(chunk)})]
            n = len(chunk)
        else:
            h, m = {}, {}
            for i, (a, b) in enumerate(chunk):
                h[2 * i], m[2 * i] = (a,), (b,)
                (h if i % 2 else m)[2 * i + 1] = (rng.randrange(256),)
            lists = [("C+h?", h), ("C+m?", m)]
            n = 2 * len(chunk)
        reads.append(Read("two_" + shape, lists, n, rev=len(reads) % 2 == 1))


def multi_lists(shape, cases):
    """Lists of a multi-code shape holding `cases` (one tuple of bytes per slot, in the order of the shape's codes)."""
    if shape in ("hmf", "hmfc"):
        return [("C+%s?" % shape, {i: c for i, c in enumerate(cases)})]
    codes = {"h_m_f": "hmf", "h_m_chebi": ["h", "m", CHEBI], "h_m_f_chebi": ["h", "m", "f", CHEBI]}[shape]
    return [("C+%s?" % c, {i: (v[j],) for i, v in enumerate(cases)}) for j, c in enumerate(codes)]


def multi_cases(rng, n_codes):
    """Byte tuples of n_codes codes on one base: canonical ties (the sum plus the largest = 254), mod-mod ties, the
    ReDistribute ties (dropped + kept + kept + 2 x one kept = 254), and random tuples whose sum stays <= 255."""
    out = set()
    while len(out) < 90:                                         # canonical ties
        v = [rng.randrange(90) for _ in range(n_codes - 1)]
        x = 254 - sum(v)
        if x % 2 == 0 and x // 2 >= max(v):
            t = v + [x // 2]
            rng.shuffle(t)
            out.add(tuple(t))
    ties = set()
    while len(ties) < 60:                                         # mod-mod ties
        a = rng.randrange(40, 128)
        v = [a, a] + [rng.randrange(0, a) for _ in range(n_codes - 2)]
        if sum(v) <= 255:
            rng.shuffle(v)
            ties.add(tuple(v))
    rd = set()
    while len(rd) < 300:                                         # ReDistribute ties: sum(v) + v[j] = 254 for a kept j
        v = [rng.randrange(100) for _ in range(n_codes)]
        j = rng.randrange(n_codes)
        rest = 254 - sum(v) - v[j]
        if rest >= 0 and rest % 2 == 0:
            v[j] += rest // 2
            if sum(v) <= 255:
                rd.add(tuple(v))
    rnd = set()
    while len(rnd) < 200:
        cut = sorted(rng.randrange(256) for _ in range(n_codes))
        rnd.add(tuple([cut[0]] + [b - a for a, b in zip(cut, cut[1:])]))
    return sorted(out) + sorted(ties) + sorted(rd) + sorted(rnd)


@functools.lru_cache(maxsize=None)
def build_table(seed=7, duplex=False, multi=True):
    """The call table; multi=False leaves out the reads with three or four codes, whose ReDistribute shares of 1/3 are off the
    1/1024 grid of the sampled-probability histogram (so an estimated threshold under --ignore fails on them)."""
    rng = random.Random(seed)
    reads = []
    grid = [(a, s - a) for s in range(0, 263) for a in range(0, min(s, 255) + 1) if s - a <= 255]
    edge = lambda ab: ab[0] == ab[1] or 253 <= sum(ab) <= 262
    for shape in ("sep", "comb", "shift"):
        # the shared-position two-list shape takes the full grid; the others every pair with a == b or a sum of 253-262
        # and a seeded fifth of the rest
        pairs = [p for p in grid if shape == "sep" or edge(p) or rng.random() < 0.2]
        ok = [p for p in pairs if shape == "comb" or sum(p) <= 258]
        if duplex:
            ok = [p for p in ok if edge(p) or rng.random() < 0.1]
        two_code_reads(rng, reads, shape, ok)
        if shape == "sep":
            # sums >= 259 fail the read: one per dedicated read, beside an identical read at 258
            for a, b in (p for p in pairs if sum(p) >= 259 and (not duplex or p[0] % 8 == 0)):
                for bb in (b, 258 - a):
                    reads.append(Read("fail_sum", [("C+h?", {0: (a,)}), ("C+m?", {0: (bb,)})], 1, rev=len(reads) % 2 == 1))
    for a, b in itertools.product(range(127, 132), repeat=2):     # the same code in two lists
        reads.append(Read("dup_code", [("C+m?", {0: (a,)}), ("C+m?", {0: (b,)})], 1, rev=len(reads) % 2 == 1))
    for shape, n_codes in (("hmf", 3), ("h_m_f", 3), ("h_m_chebi", 3), ("hmfc", 4), ("h_m_f_chebi", 4)) if multi else ():
        cases = multi_cases(rng, n_codes)
        for k in range(0, len(cases), 40):
            reads.append(Read("multi_" + shape, multi_lists(shape, cases[k:k + 40]), len(cases[k:k + 40]), rev=len(reads) % 2 == 1))
    if duplex:
        for r in reads:
            r.rev = False
            r.lists = r.lists + [("G-" + h[2:], calls) for h, calls in r.lists]
    table = Table(reads, {})
    table.thresholds = decisive_thresholds(table) if multi else {}
    return table


def write_table(table, dirpath, name="calls"):
    """BAM and FASTA of the table: forward reads end to end, then the reverse reads, each read exactly its slots' units."""
    fwd = [r for r in table.reads if not r.rev]
    rev = [r for r in table.reads if r.rev]
    seq, pos = [], 0
    for r in fwd + rev:
        r.start = pos
        seq.append(UNIT * r.n + GAP)
        pos += 4 * r.n + len(GAP)
    g = Genome(1, ct=0)
    g.contigs["ct"] = "".join(seq) + "A" * 100
    for r in table.reads:
        def heads(read, r=r):
            cs = [q for q, c in enumerate(read) if c == "C"]
            gs = [q for q, c in enumerate(read) if c == "G"]
            assert len(cs) == len(gs) == r.n
            return [(h, [((cs if h[0] == "C" else gs)[s], v if len(v) > 1 else v[0]) for s, v in sorted(calls.items())]) for h, calls in r.lists]
        g.add("ct", r.start, [("M", 4 * r.n)], rev=r.rev, seq=g.contigs["ct"][r.start:r.start + 4 * r.n], heads=heads)
    return g.write(dirpath, name)


# ---------------------------------------------------------------------------------------------------------------------------
# the model of a whole run

def parse_flags(flags):
    """(caller, ignore, combine_mods, combine_strands, percentile or None) of pileup flags."""
    per_mod, per_base, default, ignore, pct = {}, {}, None, None, 0.1
    combine_mods = combine_strands = no_filt = False
    it = iter(flags)
    for f in it:
        if f == "--no-filtering":
            no_filt = True
        elif f == "--filter-threshold":
            v = next(it)
            if ":" in v:
                per_base[v.split(":")[0]] = float(v.split(":")[1])
            else:
                default = float(v)
        elif f == "--mod-thresholds":
            k, v = next(it).split(":")
            per_mod[k] = float(v)
        elif f == "--ignore":
            ignore = next(it)
        elif f == "--preset":
            next(it)
            ignore, combine_strands = "h", True
        elif f == "--combine-mods":
            combine_mods = True
        elif f == "--combine-strands":
            combine_strands = True
        elif f == "-p":
            pct = float(next(it))
        elif f in ("--ref", "--motif", "--devices"):
            next(it)
            if f == "--motif":
                next(it)
    estimated = not no_filt and not per_base and default is None
    caller = cm.Caller(per_mod, per_base, default or 0.0)
    return caller, ignore, combine_mods, combine_strands, (pct if estimated else None)


_MODEL_RUNS = {}


def model_run(table, flags, exact=False):
    """{(position, strand): (read, call, argmax, codes)} of the surviving reads, the failed reads, and the estimated threshold
    (kept per table and flag set: the motif and the reference do not change a call)."""
    drop = set()
    for i, f in enumerate(flags):
        drop |= {i, i + 1, i + 2} if f == "--motif" else {i, i + 1} if f in ("--ref", "--devices") else set()
    key = (id(table), tuple(f for i, f in enumerate(flags) if i not in drop), exact)
    if key not in _MODEL_RUNS:
        _MODEL_RUNS[key] = _model_run(table, flags, exact)
    return _MODEL_RUNS[key]


def _model_run(table, flags, exact):
    caller, ignore, _, _, pct = parse_flags(flags)
    per_read = [(r, cm.read_calls(r.model_lists(), cm.Caller(), ignore, exact=exact)) for r in table.reads]
    thr = None
    if pct is not None:
        thr = cm.percentile([a[2] for _, res in per_read if res for _, a, _ in res.values()], pct)
        caller = cm.Caller(caller.per_mod, {"C": thr})
    calls, failed = {}, []
    for r, res in per_read:
        if res is None:
            failed.append(r)
            continue
        res = cm.read_calls(r.model_lists(), caller, ignore, exact=exact)
        for slot, (c, a, codes) in res.items():
            calls[r.position(slot)] = (r, c, a, codes)
    return calls, failed, thr


def parse_bed(text):
    rows = {}
    for line in text.splitlines():
        f = line.split()
        rows.setdefault((int(f[1]), f[5]), {})[cm.code_of(f[3])] = tuple(int(x) for x in (f[9],) + tuple(f[11:18]))
    return rows


def check_rows_against_model(text, table, flags):
    """Every row's counts are the model's call at its position; the positions with rows are the surviving reads' calls."""
    _, _, combine_mods, combine_strands, _ = parse_flags(flags)
    calls, failed, _ = model_run(table, flags)
    read_codes = {}                                         # a read has rows for every code of its table at each of its calls
    for r, c, a, codes in calls.values():
        read_codes[id(r)] = read_codes.get(id(r), frozenset()) | codes
    exp = {}
    for (pos, strand), (r, c, a, codes) in calls.items():
        if c[0] == "fail":                                  # no valid coverage, no row: a failed call shows as a missing row
            continue
        key = (pos - 1, ".") if combine_strands and strand == "-" else (pos, "." if combine_strands else strand)
        row_codes = {"C"} if combine_mods else read_codes[id(r)]
        if not row_codes:                                   # --ignore of a read's only code: canonical calls without a row
            continue
        exp[key] = {}
        for code in row_codes:
            kind, called = c[0], c[1]
            n_mod = int(kind == "mod" and (combine_mods or called == code))
            n_other = int(kind == "mod" and not n_mod)
            n_canon = int(kind == "canonical")
            exp[key][code] = (n_mod + n_other + n_canon, n_mod, n_canon, n_other, 0, 0, 0, 0)
    got = parse_bed(text)
    assert set(got) == set(exp), (len(set(got) - set(exp)), len(set(exp) - set(got)), sorted(set(got) ^ set(exp))[:5])
    bad = [(k, got[k], exp[k]) for k in exp if got[k] != exp[k]]
    assert not bad, (len(bad), bad[:5])
    return len(exp), len(failed)


# ---------------------------------------------------------------------------------------------------------------------------
# thresholds where f32 decides

def decisive_thresholds(table):
    """For each --ignore code: a threshold at the f32 value of a collapsed probability that is above its exact value (the f32
    call passes `>=`, the exact one does not), taken from the table's multi-code reads."""
    out = {}
    for ignore in ("h", "m", CHEBI):
        best = None
        for r in table.reads:
            if not r.family.startswith("multi_"):
                continue
            f = cm.read_calls(r.model_lists(), cm.Caller(), ignore)
            e = cm.read_calls(r.model_lists(), cm.Caller(), ignore, exact=True)
            for slot in f:
                if f[slot][1][0] == "mod" and e[slot][1][0] == "mod" and f[slot][1][1] == e[slot][1][1]:
                    v, x = f[slot][1][2], e[slot][1][2]
                    if cm.Fraction(float(v)) > x and (best is None or v > best):
                        best = v
        out[ignore] = best
    return out


def flag_sets(table, fa=None):
    """(id, pileup flags) of the table's runs."""
    ref = ["--ref", fa] if fa else []
    nb = lambda x, d: f32_text(np.nextafter(np.float32(x), np.float32(d)))
    t = table.thresholds
    sets = [
        ("no_filtering", ["--no-filtering"]),
        ("C_384_512", ["--filter-threshold", "C:0.75"]),
        ("C_384_512_below", ["--filter-threshold", "C:" + nb(0.75, 0)]),
        ("C_384_512_above", ["--filter-threshold", "C:" + nb(0.75, 1)]),
        ("C_513_1024", ["--filter-threshold", "C:" + f32_text(513 / 1024)]),
        ("C_513_1024_above", ["--filter-threshold", "C:" + nb(513 / 1024, 1)]),
        ("default_641_1024", ["--filter-threshold", f32_text(641 / 1024)]),
        ("mod_m", ["--mod-thresholds", "m:" + f32_text(615 / 1024), "--filter-threshold", "C:" + f32_text(301 / 512)]),
        ("mod_anymod_C", ["--mod-thresholds", "C:" + f32_text(717 / 1024), "--filter-threshold", "C:0.5"]),
        ("ignore_h", ["--ignore", "h", "--filter-threshold", "C:" + f32_text(t["h"])]),
        ("ignore_m", ["--ignore", "m", "--filter-threshold", "C:" + f32_text(t["m"])]),
        ("ignore_chebi", ["--ignore", CHEBI, "--filter-threshold", "C:" + f32_text(t[CHEBI])]),
        ("ignore_m_mod_h", ["--ignore", "m", "--mod-thresholds", "h:" + f32_text(t["m"]), "--filter-threshold", "C:0.25"]),
        ("combine_mods", ["--combine-mods", "--filter-threshold", "C:" + f32_text(307 / 512)]),
        ("estimated_p01", ["-p", "0.1"]),
        ("estimated_p05", ["-p", "0.5"]),
    ]
    if fa:
        sets.append(("traditional", ["--preset", "traditional"] + ref))
    return sets


def decisive_calls(table):
    """Calls whose f32 answer differs from the exact one, over the --ignore flag sets (multi-code and repeated-code reads)."""
    n = 0
    for _, flags in flag_sets(table):
        caller, ignore, _, _, pct = parse_flags(flags)
        if pct is not None:
            continue
        for r in table.reads:
            if not (r.family.startswith("multi_") or r.family == "dup_code"):
                continue
            f = cm.read_calls(r.model_lists(), caller, ignore)
            e = cm.read_calls(r.model_lists(), caller, ignore, exact=True)
            if (f is None) != (e is None):
                n += r.n
                continue
            n += sum(f[s][0][:2] != e[s][0][:2] for s in (f or {}))
    return n


def tie_counts(table):
    """(canonical ties, mod-mod ties) among the calls of --no-filtering: the top mod probability equals the canonical one,
    or two mod codes share the top probability (both decided by the hash order)."""
    canon = modmod = 0
    for r in table.reads:
        try:
            ms = cm.position_maps([([cm.code_of(c) for c in codes], calls) for codes, calls in r.model_lists()], cm.Arith(False))
        except cm.ReadError:
            continue
        for m in ms.values():
            ps = [p for _, p in m.items()]
            top = max(ps)
            canon += top == cm.canonical_prob(m, cm.Arith(False))
            modmod += ps.count(top) > 1
    return canon, modmod


# ---------------------------------------------------------------------------------------------------------------------------
# checks of the model

def test_model_hash_order_and_known_values():
    # bucket = code & 3 for letters in 4 buckets (h 0, m 1, f 2, c 3), 5 * code & 7 in 8 (h 0, m 1, f 6, c 7); the ChEBI code
    # takes bucket 2 in both: it probes past f in a 4-bucket table and comes before f once the 4th code grows the table
    assert cm.map_order("hm") == ["h", "m"] and cm.map_order("mh") == ["h", "m"]
    assert cm.map_order("hmf") == ["h", "m", "f"] and cm.map_order("fhm") == ["h", "m", "f"]
    assert cm.fx_hash(int(CHEBI)) & 7 == 2
    assert cm.map_order(["h", "f", int(CHEBI)]) == ["h", "f", int(CHEBI)]
    assert cm.map_order([int(CHEBI), "f", "h"]) == ["h", int(CHEBI), "f"]
    assert cm.map_order(["h", "m", "f", int(CHEBI)]) == ["h", "m", int(CHEBI), "f"]
    assert cm.map_order("hmfc") == list("hmfc") and cm.map_order("chmf") == list("hmfc")
    # the issue's arg-max above 1: C+h? 2, C+m? 255 collapsed with --ignore h
    res = cm.read_calls([(["h"], {0: (2,)}), (["m"], {0: (255,)})], cm.Caller(), "h")
    assert res[0][1] == ("mod", "m", np.float32(255.5 / 256 + 2.5 / 512)) and res[0][1][2] > 1
    # two C+m? lists of 128: one code at 1.0039, accepted (<= 1.01)
    res = cm.read_calls([(["m"], {0: (128,)}), (["m"], {0: (128,)})], cm.Caller())
    assert res[0][1][2] == np.float32(257 / 256)
    # 259 on two lists fails, 258 passes; the same bytes in one list pass
    assert cm.read_calls([(["h"], {0: (3,)}), (["m"], {0: (255,)})], cm.Caller()) is None
    assert cm.read_calls([(["h", "m"], {0: (3, 255)})], cm.Caller()) is not None
    # an exact h/m tie goes to the later code in iteration order (m); a mod/canonical tie to the canonical call
    assert cm.read_calls([(["m", "h"], {0: (100, 100)})], cm.Caller())[0][0][:2] == ("mod", "m")
    assert cm.read_calls([(list("hmf"), {0: (50, 20, 92)})], cm.Caller())[0][0][:2] == ("canonical", None)


def test_percentile_matches_reference_formula():
    xs = [cm.F32(k / 1024) for k in (5, 900, 1027, 17, 1024, 300)]
    assert cm.percentile(xs, 0.5) == cm.F32(cm.F32(cm.F32(300 / 1024) * cm.F32(0.5)) + cm.F32(cm.F32(900 / 1024) * cm.F32(0.5)))
    assert cm.percentile(xs, 1.0) == cm.F32(1027 / 1024)


def test_table_families_and_decisive_cases():
    table = build_table()
    fams = {}
    for r in table.reads:
        fams[r.family] = fams.get(r.family, 0) + r.n
    want = {"two_sep", "two_comb", "two_shift", "fail_sum", "dup_code", "multi_hmf", "multi_h_m_f", "multi_h_m_chebi",
            "multi_hmfc", "multi_h_m_f_chebi"}
    assert set(fams) == want, fams
    # every a == b and every sum 253..262 in each two-code shape (sums >= 259 of the two-list shapes on dedicated reads)
    for fam in ("two_sep", "two_comb", "two_shift"):
        seen = set()
        for r in table.reads:
            if r.family == fam or (fam == "two_sep" and r.family == "fail_sum"):
                ls = r.model_lists()
                for s in ls[0][1]:
                    v = tuple(x for _, calls in ls for x in calls.get(s, ()))
                    if len(v) == 2:
                        seen.add(v)
        assert all((a, a) in seen for a in range(128)), fam
        for s in range(253, 263 if fam != "two_shift" else 259):
            assert all((a, s - a) in seen for a in range(max(0, s - 255), min(s, 255) + 1)), (fam, s)
    dec = decisive_calls(table)
    canon, modmod = tie_counts(table)
    print("families (calls): %s; f32-decisive calls: %d; canonical ties: %d; mod-mod ties: %d; thresholds: %s"
          % (fams, dec, canon, modmod, {k: f32_text(v) for k, v in table.thresholds.items()}))
    assert all(v is not None for v in table.thresholds.values())
    assert dec >= 100 and canon >= 50 and modmod >= 50


@pytest.fixture(scope="module")
def table_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("calltable")
    table = build_table()
    bam, fa = write_table(table, d)
    return table, bam, fa


@pytest.mark.parametrize("name", [n for n, _ in flag_sets(build_table(), "FA")])
def test_model_matches_oracle_pileup(name, table_files, oracle_exe, tmp_path):
    table, bam, fa = table_files
    flags = dict(flag_sets(table, fa))[name]
    text = run_oracle(oracle_exe, flags, bam, str(tmp_path / "o.bed"))
    n_pos, n_failed = check_rows_against_model(text, table, flags)
    assert n_pos > 500 and n_failed > 900


def test_model_matches_oracle_reports(table_files, oracle_exe):
    """summary --tsv and sample-probs --no-sampling: the pass / fail counts per call and the arg-max percentiles."""
    table, bam, _ = table_files
    for flags in (["--no-filtering"], ["--filter-threshold", "C:0.75"], ["--ignore", "h", "--filter-threshold", "C:" + f32_text(table.thresholds["h"])], []):
        out = subprocess.run([oracle_exe, "summary", "--tsv", "--no-sampling"] + flags + [bam], capture_output=True, text=True, check=True).stdout
        d = dict(ln.split("\t") for ln in out.splitlines() if "\t" in ln)
        calls, _, _ = model_run(table, flags or ["-p", "0.1"])
        n_pass = {}
        for _, c, a, _ in calls.values():
            k = ("pass", c[1] or "-") if c[0] != "fail" else ("fail", a[1] or "-")
            n_pass[k] = n_pass.get(k, 0) + 1
        assert int(d["C_pass_calls_unmodified"]) == n_pass.get(("pass", "-"), 0), flags
        assert int(d["C_fail_calls_unmodified"]) == n_pass.get(("fail", "-"), 0), flags
        for key in d:                                       # codes the report lists
            if key.startswith(("C_pass_calls_modified_", "C_fail_calls_modified_")):
                pf, code = key.split("_")[1], cm.code_of(key.split("_")[-1])
                assert int(d[key]) == n_pass.get((pf, code), 0), (flags, key)
        assert int(d["C_total_mod_calls"]) == sum(v for k, v in n_pass.items() if k[0] == "pass")
        assert int(d["C_total_fail_mod_calls"]) == sum(v for k, v in n_pass.items() if k[0] == "fail")
    out = subprocess.run([oracle_exe, "sample-probs", "--no-sampling", "-p", "0.1,0.5,0.9,0.999", bam], capture_output=True, text=True, check=True).stdout
    calls, _, _ = model_run(table, ["--no-filtering"])
    vals = [a[2] for _, _, a, _ in calls.values()]
    rows = [ln.split() for ln in out.splitlines()[1:]]
    assert [np.float32(r[2]) for r in rows] == [cm.percentile(vals, q) for q in (0.1, 0.5, 0.9, 0.999)]
    assert max(vals) > 1.0


def test_duplex_table_oracle_hemi_runs(hemi_oracle_exe, tmp_path):
    table = build_table(duplex=True)
    bam, fa = write_table(table, tmp_path, "duplex")
    p = subprocess.run([hemi_oracle_exe, "pileup-hemi", "-t", "4", bam, "-r", fa, "--cpg", "--no-filtering", "-o", str(tmp_path / "h.bed")],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert open(tmp_path / "h.bed").read().count("\n") > 3000


def test_python_histogram_width_matches_header():
    import re
    import modkit_b200
    from conftest import ROOT
    text = open(os.path.join(ROOT, "include", "mkp.h")).read()
    assert int(re.search(r"#define\s+MKP_HIST_BINS\s+(\d+)", text).group(1)) == modkit_b200.HIST_BINS
    assert (modkit_b200.HIST_BINS - 1) / 1024 >= 1.01 + 1.01 / 2    # the largest arg-max: a 1.01 code plus half a dropped 1.01
