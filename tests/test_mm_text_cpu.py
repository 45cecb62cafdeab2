"""The MM text in front of the call arithmetic: a corpus of hand-built MM / ML tags (number shapes, the kernels' fast-to-exact
tokenizer switch, white space, truncated lists, u32 edges, header forms, part separators, aliased lists), each on its own
depth-1 read, so that every bedMethyl row is one read's call. This file holds the corpus the GPU suite (test_gpu_mm_text.py)
shares and the CPU checks: the independent model (mmmodel.py, composed with callmodel.py) reproduces the reference's own
unit known-answers, agrees with the oracle row for row on every flag set, and the corpus reaches what it is meant to."""
import functools
import subprocess

import pytest

import bamio
import callmodel as cm
import mmmodel as mm
from conftest import run_oracle
from test_call_table_cpu import parse_bed
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)

GAP = "TT"


def cgat(n):
    """n units CGAT: the k-th C at 4k (a CpG), G, A and T beside it."""
    return "CGAT" * n


def poly_c(n):
    return "C" * n + "GG"


def digits(n_tokens, first="0"):
    return ",".join([first] + ["0"] * (n_tokens - 1)) if n_tokens else ""


def fill(nbytes):
    """Exactly nbytes of `0,` tokens (one `00,` when odd); nbytes >= 2, or 0."""
    assert nbytes == 0 or nbytes >= 2
    return ("00," if nbytes & 1 else "") + "0," * ((nbytes - 3 * (nbytes & 1)) // 2)


def ml_bytes(n, mod=256):
    """n ML bytes, distinct within any run of `mod`, a mix of modified and canonical calls."""
    return [(i * 53 + 11) % mod for i in range(n)]


class Case:
    """One corpus read: the forward read's bases, MM bytes, ML bytes, orientation; `pad` shifts the MM start in the packed
    block (the read grows by 2 pad bases)."""

    def __init__(self, family, read, mm_text, ml, rev, pad, note):
        self.family, self.read, self.mm, self.ml, self.rev, self.pad, self.note = family, read, mm_text, ml, rev, pad, note
        self.start = None

    @functools.cached_property
    def tables(self):
        """The model's tables, or None when the read fails."""
        try:
            return mm.mod_base_info(self.mm, self.ml, self.read)
        except cm.ReadError:
            return None

    @property
    def mm_align(self):
        """Address of the MM text modulo 4 in the packed block (16-byte aligned): one CIGAR word, the packed SEQ, the ML bytes."""
        return (4 + (len(self.read) + 1) // 2 + len(self.ml)) & 3

    def delta_texts(self):
        """[(offset in the MM text, delta text)] of the parts that have a header comma."""
        out, off = [], 0
        for part in self.mm.split(b";"):
            if b"," in part:
                k = part.index(b",") + 1
                out.append((off + k, part[k:]))
            off += len(part) + 1
        return out


class Corpus:
    def __init__(self):
        self.cases = []

    def add(self, family, text, n_ml, read=None, variants=8, ml_mod=256, note=None, sweep=None):
        """`text` (str, bytes or a function of the padded read) on `variants` reads: both orientations times four paddings of
        the read (which shift the MM start) for 8, one or two combinations picked in rotation for 1 or 2. n_ml: the ML length,
        or the bytes. sweep=o (a text that moves a byte through the offsets o): four reads, padded so that the MM text starts at
        each of the four addresses modulo 4, the orientation alternating so that every alignment sees both."""
        read = cgat(40) if read is None else read
        combos = range(8) if variants == 8 else [(len(self.cases) + 5 * j) % 8 for j in range(variants)]
        if sweep is not None:
            n = len(n_ml) if isinstance(n_ml, (list, tuple)) else n_ml
            pads = [(a - (4 + (len(read) + 1) // 2 + n)) & 3 for a in range(4)]
            combos = [2 * pad + (((sweep >> 2) + a) & 1) for a, pad in enumerate(pads)]
        for k in combos:
            r = read + "TA" * (k >> 1)
            t = text(r) if callable(text) else text
            t = t.encode("latin-1") if isinstance(t, str) else t
            ml = list(n_ml) if isinstance(n_ml, (list, tuple)) else ml_bytes(n_ml, ml_mod)
            self.cases.append(Case(family, r, t, ml, bool(k & 1), k >> 1, note))


def n_tokens(text):
    return text.count(",") + 1


@functools.lru_cache(maxsize=None)
def build_corpus(duplex=False):
    c = Corpus()
    C500 = poly_c(700)
    # ---- numbers the fast path takes: every digit count, powers of ten and their neighbours, zero padding ----------------
    for d in range(1, 10):
        c.add("numbers", "C+m?,%s,%s,0" % ("0" * (d - 1) + "3", "0" * d), 3)
    big = [9, 10, 11, 99, 100, 101, 999, 1000, 1001, 9999, 10000, 10001]
    c.add("numbers", "C+m?," + ",".join(map(str, big)), len(big), read=poly_c(sum(big) + len(big)), variants=1)
    c.add("numbers", "C+m?," + ",".join(map(str, big)), len(big), read=poly_c(sum(big) + len(big) - 1), variants=1)   # one C short
    for v in (99999, 100000, 999999999, 123456789):              # parsed by the fast path, then past the read's end
        c.add("numbers", "C+m?,1,%d,2" % v, 3)
    for o in range(128):                                         # a 9-digit number starting at every offset modulo 128
        c.add("numbers", "C+m?," + fill(123 + o) + "000000012,0,0,1", n_tokens(fill(123 + o)) + 3, read=C500, sweep=o, note=("number", 128 + o))
    c.add("numbers", "C+m?," + digits(3100), 3100, read=poly_c(3100), variants=2)
    for n in (31, 32, 33, 64, 65, 95, 96, 97, 128, 129, 159, 160, 161):
        c.add("numbers", "C+m?," + digits(n, "1"), n, read=C500)
    # ---- the fast path gives up: a 10th digit after tokens were placed, tokens longer than a round and than the staging ----
    for n, at in ((40, 0), (40, 1), (40, 32), (40, 39), (100, 70), (600, 580), (600, 599)):
        toks = ["0"] * n
        toks[at] = "0000000001"
        c.add("switch", "C+m?," + ",".join(toks), n, read=C500 + C500)
    for n in (20, 33, 127, 128, 129, 161, 300):
        c.add("switch", "C+m?,1," + "0" * (n - 1) + "2,3", 3)
        c.add("switch", "C+m?," + "0" * (n - 1) + "2", 1, variants=2)
    for o in range(128):                                         # the switch at every offset modulo 128
        c.add("switch", "C+m?," + fill(123 + o) + "0000000001,0,1", n_tokens(fill(123 + o)) + 2, read=C500, sweep=o, note=("switch", 128 + o))
    # ---- white space: space, tab, CR, LF are skipped around a number; VT and FF are not white space ---------------------------
    for w in " \t\r\n\x0b\x0c":
        for t in ("1,%s2,3", "1,2%s,3", "%s1,2,3", "1,2,3%s", "1,%s,3", "1%s2,3", "%s", "1,2%s%s3"):
            c.add("white_space", "C+m?," + t.replace("%s", w) + ";A+a?,0,1", 5)
    c.add("white_space", "C+m?, 1 ,\t2\t,\r3\r,\n4\n, \t\r\n5 \t\r\n;A+a?,0", 6)
    for run in (1, 2, 3, 5, 8, 16, 33, 40):                       # runs across the round edge (128) and the staging edge (160)
        for edge in (132, 164, 260, 292):
            pre = fill(edge - 5 - (run + 1) // 2)
            for w in (" ", "\t \r\n"):
                ws = (w * run)[:run]
                c.add("white_space", "C+m?," + pre + ws + "1" + ws + ",0,2", n_tokens(pre) + 2, read=C500, variants=1)
    # ---- truncation: the list ends at its first malformed token; the rest of the part is dropped; ML is then read shifted ------
    for bad, included in (("", 0), ("x", 0), ("-2", 0), ("+2", 0), ("2.5", 1), ("0x3", 1), ("2 3", 1), ("\x0b1", 0)):
        for at in (0, 1, 31, 32, 33, 200):
            toks = ["0"] * at + [bad, "0", "1"]
            text = "C+m?," + ",".join(toks) + ";A+a?,0,1,0"
            kept, full = at + included, len(toks)
            for n_ml in (kept + 3, full + 3, kept + 2):
                c.add("truncation", text, n_ml, read=cgat(300), variants=2 if at > 1 else 8, note=("truncated", kept, full))
    c.add("truncation", "C+m?,1,2,;A+a?,0", 3)
    c.add("truncation", "C+m?,1,2,;A+a?,0", 2)
    # ---- u32 edges -------------------------------------------------------------------------------------------------------------
    for v in ("4294967295", "4294967296", "1234567890123456789012345"):
        for t in ("%s", "0,%s", "0,1,%s,0", "0,%sx,1", "0,x,%s", "0,1 1,%s", " %s", "0,%s ", "0,0000%s"):
            for base, code in (("C", "m"), ("N", "n")):
                c.add("u32", "%s+%s?,%s" % (base, code, t % v), 4, variants=2)
    for extra in (-1, 0, 1):
        c.add("u32", lambda r, e=extra: "C+m?,%d" % (r.count("C") - 1 + e), 1)
        c.add("u32", lambda r, e=extra: "C+m?,0,%d" % (r.count("C") - 2 + e), 2)
        c.add("u32", lambda r, e=extra: "N+n?,%d" % (len(r) - 1 + e), 1)
        c.add("u32", lambda r, e=extra: "N+n?,0,%d" % (len(r) - 2 + e), 2)
        c.add("u32", lambda r, e=extra: "T+t?,%d;U+u?,%d" % (r.count("T") - 1, r.count("T") - 1 + e), 2)
    # ---- headers ---------------------------------------------------------------------------------------------------------------
    for b in "ACGTUNacgtnXB*":
        c.add("headers", "%s+x?,0,1" % b, 2, variants=2)
    for h in ("C+m?", "C-m?", "C*m?", "Cm?", "C+hm?", "C+?m", "C+m?.", "C+m.?", "C+m", "C+m.", "C+h?m?", "C+h.m", "C+21839?", "C+021839?",
              "C+2147483647?", "C+2147483648?", "C+2147483649?", "C+4294967295?", "C+4294967296?", "C+99999999999999999999?",
              "C+21839m?", "C+m1?", "C+21839.", "C+21839", "C+", "C+?", "C+.", "C", "+m?", " C+m?", "C +m?", "C+m_?", "C+hmfc?", "C+\xc2\xbb?",
              "C+m?\xc2\xac", "G-h?", "G-hm."):
        c.add("headers", h + ",0,1", 8, variants=2, ml_mod=64)
        c.add("headers", h + ",0,1;A+a?,0", 9, variants=2, ml_mod=64)
    for h in ("C+m?", "C+m.", "C+m", "C+hm", "C+21839", "C+", "C", "C+?"):          # no header comma: no deltas
        c.add("headers", h, 0, variants=2)
        c.add("headers", h + ";A+a?,0,1", 2, variants=2)
        c.add("headers", h + ",", 1, variants=2)
        c.add("headers", h + ",;A+a?,0", 1, variants=2)
    # ---- parts -----------------------------------------------------------------------------------------------------------------
    for t in (";C+m?,0,1", "C+m?,0,1;;A+a?,0", "C+m?,0,1;A+a?,0;", "C+m?,0,1;A+a?,0;;;", ";;C+m?,0,1;", ";", ";;", "", "C+m?,0,1;,;", "C+m?,0,1;x"):
        c.add("parts", t, 3)
    for o in range(128):                                         # a `;` and the next header comma at every offset modulo 128
        c.add("parts", "C+m?," + fill(122 + o) + "1;A+a?,2,1;T+t?,0", n_tokens(fill(122 + o)) + 3, read=C500 + cgat(5), sweep=o,
              note=("semicolon", 128 + o))
    c.add("parts", "".join("C+m?,0;" for _ in range(16)), list(range(16)))
    c.add("parts", "".join("%s+%s?,%d;" % ("CAGT"[k & 3], "mahgtxyz"[k >> 1], k >> 2) for k in range(16)), 16, ml_mod=64)
    for tail in ("x\xc2\xbb\xc2\xac,5", "\xc2\xbb,5", " \xc2\xac5,5"):    # bytes 0xBB and 0xAC are neither `;` nor `,`
        c.add("parts", "C+m?,0,1" + tail + ";A+a?,0,1", 4)
        c.add("parts", "C+m?,0," + fill(118) + "1" + tail + ",7;A+a?,0,1", n_tokens(fill(118)) + 3, read=C500 + cgat(3))
    # ---- aliases: a list whose delta text repeats the previous list's shares its entries ------------------------------------------
    def text_of(n):
        return "0" if n == 1 else (fill(n - 1) + "0")
    R = cgat(520)
    for n in (1, 3, 127, 128, 129, 1000):
        t = text_of(n)
        k = n_tokens(t)
        c.add("aliases", "C+h?,%s;C+m?,%s" % (t, t), 2 * k, read=R, ml_mod=128)
        c.add("aliases", "C+h?,%s;C+m?,%s;C+f?,%s" % (t, t, t), 3 * k, read=R, ml_mod=80, variants=2)
        c.add("aliases", "C+h?,%s;A+a?,%s" % (t, t), 2 * k, read=R, variants=2)
        c.add("aliases", "C+hm?,%s;C+f?,%s" % (t, t), 3 * k, read=R, ml_mod=80, variants=2)
        for o in sorted(set([0, n - 1] + list(range(127, n, 128)) + list(range(128, n, 128)))):
            o -= t[o] == ","
            u = t[:o] + "1" + t[o + 1:]
            c.add("aliases", "C+h?,%s;C+m?,%s" % (t, u), 2 * k, read=R, ml_mod=128, variants=2)
            c.add("aliases", "C+h?,%s;C+m?,%s" % (u, t), 2 * k, read=R, ml_mod=128, variants=2)
    for t in ("0, 1,2", "0,1,x,5", "0,1 ,2x,9", "0,0000000001,2", "0,1,"):
        c.add("aliases", "C+h?,%s;C+m?,%s" % (t, t), 6, ml_mod=128)
        c.add("aliases", "C+h?,%s;C+m?,%s" % (t, t), 5, ml_mod=128, variants=2)
    if duplex:                                                   # the forward reads, each with a G- list behind its text
        c.cases = [x for x in c.cases if not x.rev and len([p for p in x.mm.split(b";") if p]) < 16]   # (16 lists per read is the device limit)
        for x in c.cases:
            x.mm = x.mm + (b"" if x.mm.endswith(b";") or not x.mm else b";") + b"G-m?,0,1;"
            x.ml = x.ml + [200, 30]
    return c


def write_corpus(corpus, dirpath, name="mmtext"):
    """BAM and FASTA: the reads end to end at depth 1, every read all-M on its own stretch of the contig."""
    pos, seq, recs = 0, [], []
    for k, x in enumerate(corpus.cases):
        stored = bamio.revcomp(x.read) if x.rev else x.read
        x.start = pos
        seq.append(stored + GAP)
        recs.append(bamio.make_record(0, pos, 16 if x.rev else 0, [("M", len(stored))], stored, name="m%d" % k,
                                      aux=(bamio.aux_z("MM", x.mm), bamio.aux_b("ML", "C", x.ml))))
        pos += len(stored) + len(GAP)
    contig = "".join(seq) + "A" * 100
    bam, fa = "%s/%s.bam" % (dirpath, name), "%s/%s.fa" % (dirpath, name)
    bamio.bam_of([("ct", len(contig))], recs).write(bam, index=True)
    bamio.write_fasta(fa, {"ct": contig})
    return bam, fa, contig


# ---------------------------------------------------------------------------------------------------------------------------
# the model of a whole run

COMP = {"A": "T", "C": "G", "G": "C", "T": "A"}


def table_calls(x, ignore=None, force=False):
    """[(strand, base, {forward position: (call, codes)})] of one read's tables under --no-filtering, inferred positions
    included, or None when the read is not used (it fails, or has a mode-less list without --force-allow-implicit)."""
    if x.tables is None:
        return None
    if any(t.mode == mm.DEFAULT for t in x.tables.values()) and not force:       # read_cache.rs:122-137
        return None
    ar, caller, out = cm.Arith(False), cm.Caller(), []
    for (strand, base), t in x.tables.items():
        tb = base if strand == "+" else COMP[base]
        res = cm.read_calls([([str(c) for c in codes], v) for codes, v in t.lists], caller, ignore, base=tb) if t.lists else {}
        if res is None:
            return None
        calls = {p: (call, codes) for p, (call, _, codes) in res.items()}
        for p, codes in t.inferred.items():
            m = cm.FxMap(reserve=len(codes))
            for code in codes:
                m.insert(code, ar.num(0.0))
            if ignore is not None:
                m = cm.redistribute(m, cm.code_of(ignore), ar)
            calls[p] = (cm.call(m, caller, tb, ar), frozenset(k for k, _ in m.items()))
        out.append((strand, base, calls))
    return out


def read_rows(x, ignore=None, combine_mods=False, force=False):
    """{(reference position, strand): {code: counts}} of one read under --no-filtering, or None when the read is not used."""
    tables = table_calls(x, ignore, force)
    if tables is None:
        return None
    rows = {}
    for strand, base, calls in tables:
        tb = base if strand == "+" else COMP[base]
        all_codes = frozenset().union(*(codes for _, codes in calls.values())) if calls else frozenset()
        row_codes = {tb} if combine_mods else all_codes
        ref_strand = "+" if (strand == "+") != x.rev else "-"
        for p, (call, _) in calls.items():
            q = len(x.read) - 1 - p if x.rev else p
            for code in row_codes:
                n_mod = int(call[0] == "mod" and (combine_mods or call[1] == code))
                n_other = int(call[0] == "mod" and not n_mod)
                n_canon = int(call[0] == "canonical")
                rows.setdefault((x.start + q, ref_strand), {})[code] = (1, n_mod, n_canon, n_other, 0, 0, 0, 0)
    return rows


def summary_totals(corpus, ignore=None):
    """What `summary --no-sampling --no-filtering --tsv` reports, from the model: {key: count} of the reads used, the reads per
    base and the calls per base and code. The sampler takes mode-less lists as they are; a `-` strand table is reported under the complement of its base."""
    out = {"total_reads_used": 0}
    for x in corpus.cases:
        tables = table_calls(x, ignore, force=True)
        if not tables:
            continue
        out["total_reads_used"] += 1
        tables = [(strand, base if strand == "+" else COMP[base], calls) for strand, base, calls in tables]
        for base in {b for _, b, _ in tables}:
            out["count_reads_" + base] = out.get("count_reads_" + base, 0) + 1
        for _, base, calls in tables:
            for call, _ in calls.values():
                key = "%s_pass_calls_%s" % (base, "unmodified" if call[0] == "canonical" else "modified_%s" % call[1])
                out[key] = out.get(key, 0) + 1
                out[base + "_total_mod_calls"] = out.get(base + "_total_mod_calls", 0) + 1
    return out


def check_summary(text, corpus, ignore=None):
    """Every count of a `summary --tsv` text against the model's totals."""
    got = {k: int(v) for k, v in (ln.split("\t") for ln in text.splitlines() if "\t" in ln) if v.isdigit() and "_frac_" not in k}
    exp = summary_totals(corpus, ignore)
    bad = {k: (got.get(k), exp.get(k, 0)) for k in set(got) | set(exp) if got.get(k, 0) != exp.get(k, 0)}
    assert not bad, bad
    return exp["total_reads_used"]


def parse_flags(flags):
    ignore = flags[flags.index("--ignore") + 1] if "--ignore" in flags else None
    return dict(ignore=ignore, combine_mods="--combine-mods" in flags, force="--force-allow-implicit" in flags)


def model_rows(corpus, contig, flags):
    """(expected rows, used reads, unused reads) of a pileup run; --cpg keeps the CpG positions of either strand."""
    exp, used, unused, cut = {}, 0, 0, 0
    for x in corpus.cases:
        rows = read_rows(x, **parse_flags(flags))
        if rows is None:
            unused += 1
            continue
        used += 1
        for (pos, strand), v in rows.items():
            c_pos = pos if strand == "+" else pos - 1                   # the C of the CpG on the + strand
            if "--cpg" in flags and not (c_pos >= 0 and contig[c_pos:c_pos + 2] == "CG" and c_pos // INTERVAL == (c_pos + 1) // INTERVAL):
                cut += c_pos >= 0 and contig[c_pos:c_pos + 2] == "CG"
                continue
            assert (pos, strand) not in exp
            exp[(pos, strand)] = v
    assert "--cpg" not in flags or cut >= 1                          # the corpus keeps a call on a CpG cut by an interval boundary
    return exp, used, unused


def check_rows(text, corpus, contig, flags):
    exp, used, unused = model_rows(corpus, contig, flags)
    got = parse_bed(text)
    by_start = sorted((x.start, k) for k, x in enumerate(corpus.cases))

    def case_of(pos):
        import bisect
        x = corpus.cases[by_start[bisect.bisect_right(by_start, (pos, 1 << 60)) - 1][1]]
        return (x.family, x.mm[:60], len(x.ml), x.rev, x.pad)
    diff = sorted(set(got) ^ set(exp))
    assert not diff, (len(diff), [(k, "extra" if k in got else "missing", case_of(k[0])) for k in diff[:4]])
    bad = [(k, got[k], exp[k], case_of(k[0])) for k in exp if got[k] != exp[k]]
    assert not bad, (len(bad), bad[:4])
    return len(exp), used, unused


INTERVAL = 100000            # --interval-size: motifs are searched per interval (fasta.rs:208-225), so a CpG whose two bases lie in
                             # different intervals is not a motif position, in the reference as here
FLAG_SETS = [
    ("all", ["--no-filtering"]),
    ("all_force", ["--no-filtering", "--force-allow-implicit"]),
    ("cpg", ["--no-filtering", "--cpg", "--ref", "FA"]),
    ("cpg_force", ["--no-filtering", "--cpg", "--ref", "FA", "--force-allow-implicit"]),
    ("ignore_h", ["--no-filtering", "--ignore", "h"]),
    ("combine_mods", ["--no-filtering", "--combine-mods", "--force-allow-implicit"]),
]


# ---------------------------------------------------------------------------------------------------------------------------
# the model against the reference's own known answers

def test_model_parse_known_answers():
    for text, mode in (("C+h?", mm.EXPLICIT), ("C+m", mm.DEFAULT), ("C+m.", mm.IMPLICIT)):      # mod_bam.rs:2193-2227
        got = mm.parse_part((text + ",5,2,1,3,1,2,3,1,2,1,11,5").encode())
        assert got == mm.MmList("C", "+", mode, [text[2]], [5, 2, 1, 3, 1, 2, 3, 1, 2, 1, 11, 5])
    lists = mm.parse_mm_tag(b"C+h?,1,1,0;C+m?,1,1,0;G-h?,1,2,0;G-m?,1,2,0")                 # :2515
    assert [(x.base, x.strand, x.codes, x.deltas) for x in lists][2:] == [("G", "-", ["h"], [1, 2, 0]), ("G", "-", ["m"], [1, 2, 0])]
    assert [x.deltas for x in mm.parse_mm_tag(b"C+h?;C+m?;")] == [[], []]                       # :2709
    # nom: white space is space, tab, CR, LF; the list ends before the separator whose element fails
    assert mm.parse_int_list(b" 1 ,\t2\r\n,3") == [1, 2, 3]
    assert mm.parse_int_list(b"1,,2") == [1] and mm.parse_int_list(b"1,2,") == [1, 2] and mm.parse_int_list(b"1,x,3") == [1]
    assert mm.parse_int_list(b"1,2.5,7") == [1, 2] and mm.parse_int_list(b"1 2,3") == [1] and mm.parse_int_list(b"1,\x0b2") == [1]
    assert mm.parse_int_list(b"4294967295") == [4294967295] and mm.parse_int_list(b"1,x,4294967296") == [1]
    for bad in (b"", b",1", b"x", b"\x0c1", b"4294967296", b"1,4294967296", b"1,4294967296x"):
        with pytest.raises(cm.ReadError):
            mm.parse_int_list(bad)
    # header forms: the last mode character wins and may stand before a code; a ChEBI number takes no letters
    p = lambda t: mm.parse_part(t.encode("latin-1"))
    assert (p("C+?m,0").mode, p("C+?m,0").codes) == (mm.EXPLICIT, ["m"]) and p("C+m?.,0").mode == mm.IMPLICIT and p("C+m.?,0").mode == mm.EXPLICIT
    assert p("C+021839?,0").codes == [21839] and p("C+2147483647?,0").codes == [2147483647] and p("C+h?m?,0").codes == ["h", "m"]
    assert p("C+m?").deltas == [] and p("C+m").mode == mm.DEFAULT
    for bad in ("C+m?,", "C+21839m?,0", "C+m1?,0", "C+?,0", "C+", "C", "+m?,0", " C+m?,0", "c+m?,0", "C*m?,0", "C+2147483648?,0",
                "C+4294967296?,0", "C+\xbb?,0"):
        with pytest.raises(cm.ReadError):
            p(bad)


def test_model_positions_known_answers():
    seq = "ACCGCCGTCGTCG"                                                                       # mod_bam.rs:1924-1954
    for deltas, expected in (([1, 1, 0], [2, 5, 8]), ([3, 0, 0], [5, 8, 11]), ([3, 1], [5, 11])):
        assert mm.to_positions("C", deltas, seq) == expected
    dna = "GCGGATTTCTGAGTTTG"                                                                   # :2776-2785
    assert mm.to_positions("N", [5, 0, 0, 1, 3, 0, 0], dna) == [5, 6, 7, 9, 13, 14, 15]
    assert mm.to_positions("N", [len(dna)], dna) == [len(dna)]          # the first N delta is not checked here ...
    with pytest.raises(cm.ReadError):
        mm.mod_base_info(b"N+n?,%d" % len(dna), [1], dna)               # ... the reference then indexes past the end
    for base, deltas in (("C", [0, 1, 0, 5]), ("C", [4294967295]), ("C", [0, 4294967295]), ("N", [0, len(dna) - 1]), ("U", [7])):
        with pytest.raises(cm.ReadError):
            mm.to_positions(base, deltas, "GATCGACTACGTCGA" if base == "C" else dna)
    assert mm.to_positions("U", [6], dna) == [15]


def test_model_tables_known_answers():
    dna = "GATCGACTACGTCGA"                                                                     # mod_bam.rs:2230-2326
    a = mm.mod_base_info(b"C+hm?,0,1,0;", [1, 200, 1, 200, 1, 200], dna)
    b = mm.mod_base_info(b"C+h?,0,1,0;C+m?,0,1,0;", [1, 1, 1, 200, 200, 200], dna)
    assert a[("+", "C")].lists == [(["h", "m"], {3: (1, 200), 9: (1, 200), 12: (1, 200)})]
    assert b[("+", "C")].lists == [(["h"], {3: (1,), 9: (1,), 12: (1,)}), (["m"], {3: (200,), 9: (200,), 12: (200,)})]
    t = mm.mod_base_info(b"C+h?,0,1,0;A+a?,0,1,0;C+m?,0,1,0;", [1, 1, 1, 200, 200, 200, 1, 1, 1], dna)
    assert t[("+", "A")].lists == [(["a"], {1: (200,), 8: (200,), 14: (200,)})] and len(t[("+", "C")].lists) == 2
    for tag, ml in ((b"C+m?,0,1,0,5;", [1, 2, 3, 4]), (b"C+m?,0,1,0;", [1, 2])):               # past the last C; ML too short
        with pytest.raises(cm.ReadError):
            mm.mod_base_info(tag, ml, dna)
    assert mm.mod_base_info(b"C+m?,0,1,0;", [1, 2, 3, 4, 5], dna)[("+", "C")].lists[0][1][12] == (3,)     # surplus ML is ignored
    assert mm.mod_base_info(b"C+h?;C+m?;", [], dna) == {}                                       # :2706-2714
    t = mm.mod_base_info(b"C+m.,1;", [200], dna)                                                # :1265-1292
    assert sorted(t[("+", "C")].inferred) == [3, 9, 12] and t[("+", "C")].lists == [(["m"], {6: (200,)})]
    assert sorted(mm.mod_base_info(b"C+h.;C+m.;", [], dna)[("+", "C")].inferred) == [3, 6, 9, 12]
    t = mm.mod_base_info(b"N+n?,0,2;", [10, 20], dna)                                           # tables are keyed by the actual base
    assert t[("+", "G")].lists == [(["n"], {0: (10,)})] and t[("+", "C")].lists == [(["n"], {3: (20,)})]
    dna = "GCGGATTTCTGAGTTTG"                                                                   # :2828-2884
    with pytest.raises(cm.ReadError):
        mm.mod_base_info(b"C+m.;N+b?,1,3,0,0,1,3,0,0;", [255] * 8, dna)
    t = mm.mod_base_info(b"N+b?,1,3,0,0,1,3,0,0;C+m?,0;", [255] * 9, dna)
    assert cm.read_calls([([str(k) for k in codes], v) for codes, v in t[("+", "C")].lists], cm.Caller()) is None
    assert mm.mod_base_info(b"N+b?,0,1;C+m.,0,1;", [200, 255, 50, 0], "CATCACA")[("+", "C")].mode == mm.IMPLICIT
    with pytest.raises(cm.ReadError):
        mm.mod_base_info(b"C+mh.,0,1;C+h.,0", [200, 0, 0, 200, 25], "CATCACA")
    with pytest.raises(cm.ReadError):
        mm.mod_base_info(b"N+n?,0", [9], "NACGT")                                               # DnaBase::try_from


def test_fast_path_predicate():
    assert mm.fast_path(b"0") and mm.fast_path(b"123456789,0,000000000")
    for t in (b"", b"1234567890", b"1,,2", b",1", b"1,", b"1, 2", b"1,x", b"1\x0b"):
        assert not mm.fast_path(t)


# ---------------------------------------------------------------------------------------------------------------------------
# the corpus

def fused_route(x):
    """Where the fused kernel takes a read whose headers parse (mkp_fused.cuh): "single" / "alias" stay on it (per base one list of
    at most two different codes, or one list and, right behind it, a byte-identical copy of its delta text with another
    single code; `+` strand, `?` mode, no N list); "shape" leaves before tokenising, "not_alias" after it."""
    parts = [p for p in x.mm.split(b";") if p]
    lists = [mm.parse_part(p.split(b",")[0]) for p in parts]
    by_base, kind = {}, "single"
    for k, h in enumerate(lists):
        if h.base == "N" or h.strand != "+" or h.mode != mm.EXPLICIT:
            return "shape"
        by_base.setdefault("T" if h.base == "U" else h.base, []).append(k)
    for ks in by_base.values():
        h = lists[ks[0]]
        if len(ks) == 1:
            if len(h.codes) > 2 or len(set(h.codes)) != len(h.codes):
                return "shape"
        elif len(ks) > 2 or ks[1] != ks[0] + 1 or len(h.codes) != 1 or len(lists[ks[1]].codes) != 1 or h.codes == lists[ks[1]].codes:
            return "shape"
        else:
            t0, t1 = (parts[k].partition(b",") for k in ks)
            kind = "alias" if kind != "not_alias" and t0[1] and t1[1] and t0[2] == t1[2] and t0[2] else "not_alias"
    return kind


def test_corpus_reaches_the_fused_kernel_and_the_generic_one():
    routes = {}
    for x in build_corpus().cases:
        try:
            r = fused_route(x)
        except cm.ReadError:
            continue
        routes[r] = routes.get(r, 0) + 1
    print(routes)
    assert routes["single"] >= 100 and routes["alias"] >= 30 and routes["shape"] >= 100 and routes["not_alias"] >= 30, routes


def test_corpus_census():
    """Offsets are counted where the kernels see them: the list scan's rounds of 128 bytes start at the 4-aligned address at or
    below the MM text, the fast tokenizer's at the 4-aligned address at or below the delta text."""
    corpus = build_corpus()
    fams, accepted, rejected, fast, exact = {}, 0, 0, 0, 0
    hits = {k: set() for k in ("semicolon", "comma", "number", "nine_digits", "switch")}
    phases = {k: set() for k in ("semicolon", "number", "switch")}     # (MM address modulo 4, orientation) of the sweep reads
    shifted = 0
    for x in corpus.cases:
        fams[x.family] = fams.get(x.family, 0) + 1
        accepted += x.tables is not None
        rejected += x.tables is None
        a = x.mm_align
        for off, text in x.delta_texts():
            fast += mm.fast_path(text)
            exact += not mm.fast_path(text)
            hits["comma"].add((off - 1 + a) % 128)
            in_round = lambda g, off=off: (g - off + ((a + off) & 3)) % 128
            tok = off
            for t in text.split(b","):
                if t[:1].isdigit():
                    hits["number"].add(in_round(tok))
                    if len(t) == 9 and t.isdigit():
                        hits["nine_digits"].add(in_round(tok))
                tok += len(t) + 1
            if x.note and x.note[0] == "switch" and off == 5:
                assert not mm.fast_path(text) and mm.fast_path(text[:x.note[1] - off + 9])
                hits["switch"].add(in_round(x.note[1] + 9))       # the 10th digit
        for k, ch in enumerate(x.mm):
            if ch == 0x3b:
                hits["semicolon"].add((k + a) % 128)
        if x.note and x.note[0] in phases:
            phases[x.note[0]].add((a, x.rev))
        if x.note and x.note[0] == "truncated" and x.tables and len(x.tables) == 2 and len(x.ml) >= x.note[2] + 3 and x.note[1] < x.note[2]:
            shifted += 1                                         # the A list's bytes would be other bytes had the C list gone on
    print("reads %d: %s; accepted %d rejected %d; delta texts fast %d exact %d; shifted %d" % (len(corpus.cases), fams, accepted, rejected, fast, exact, shifted))
    assert set(fams) == {"numbers", "switch", "white_space", "truncation", "u32", "headers", "parts", "aliases"} and min(fams.values()) >= 150
    assert len(corpus.cases) < 5000 and accepted >= 200 and rejected >= 100 and fast >= 150 and exact >= 150
    assert all(len(v) == 128 for v in hits.values()), {k: len(v) for k, v in hits.items()}
    assert all(len(v) == 8 for v in phases.values()), phases
    assert shifted >= 30
    assert {x.pad for x in corpus.cases} == {0, 1, 2, 3} and {x.rev for x in corpus.cases} == {False, True}
    assert {(x.mm_align, x.rev) for x in corpus.cases} == {(a, r) for a in range(4) for r in (False, True)}


def test_corpus_holds_the_malformed_tag_mutations():
    """The ten mutations test_gpu_malformed_mm_tags applies to a fixture's reads, each as a corpus text of its own."""
    texts = {x.mm for x in build_corpus().cases}
    for t in (b"C+m?, 1 ,\t2\t,\r3\r,\n4\n, \t\r\n5 \t\r\n;A+a?,0", b"C+m?,0,x,0,1;A+a?,0,1,0", b"C+m?,;A+a?,0", b"C+m?;A+a?,0,1", b"C+m?,1,999999999,2",
              b"X+x?,0,1", b"C+m,0,1", b"C+21839?,0,1", b"C+m1?,0,1", b"C+m?,0,1;A+a?,0;;;"):
        assert t in texts, t


@pytest.fixture(scope="module")
def corpus_files(tmp_path_factory):
    corpus = build_corpus()
    bam, fa, contig = write_corpus(corpus, tmp_path_factory.mktemp("mmtext"))
    return corpus, bam, fa, contig


@pytest.mark.parametrize("name", [n for n, _ in FLAG_SETS])
def test_model_matches_oracle_pileup(name, corpus_files, oracle_exe, tmp_path):
    corpus, bam, fa, contig = corpus_files
    flags = [fa if f == "FA" else f for f in dict(FLAG_SETS)[name]]
    text = run_oracle(oracle_exe, flags, bam, str(tmp_path / "o.bed"))
    n_rows, used, unused = check_rows(text, corpus, contig, flags)
    print(name, n_rows, used, unused)
    assert n_rows > (300 if "--cpg" in flags else 3000) and used >= 200 and unused >= 100


def test_chebi_code_above_31_bits_is_a_read_error(oracle_exe, tmp_path):
    """`C+2147483649?` must not come out as code 1: the code representation keeps bit 31 as its ChEBI tag."""
    c = Corpus()
    for h in ("C+2147483649?", "C+4294967295?", "C+2147483647?", "C+1?"):
        c.add("chebi", h + ",0,1", 2, variants=2)
    bam, fa, contig = write_corpus(c, tmp_path, "chebi")
    text = run_oracle(oracle_exe, ["--no-filtering"], bam, str(tmp_path / "o.bed"))
    assert check_rows(text, c, contig, ["--no-filtering"])[1:] == (4, 4)
    assert {ln.split()[3] for ln in text.splitlines()} == {"2147483647", "1"}


def test_duplex_corpus_oracle_hemi_runs(hemi_oracle_exe, tmp_path):
    """The duplex variant (the forward reads, a G- list behind every text) through the hemi oracle: a failed read is one NoCall."""
    bam, fa, _ = write_corpus(build_corpus(duplex=True), tmp_path, "duplex")
    p = subprocess.run([hemi_oracle_exe, "pileup-hemi", "-t", "4", bam, "-r", fa, "--cpg", "--no-filtering", "-o", str(tmp_path / "h.bed")],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert open(tmp_path / "h.bed").read().count("\n") > 200


@pytest.mark.parametrize("ignore", [None, "h"])
def test_model_matches_oracle_summary(ignore, corpus_files, oracle_exe):
    corpus, bam, _, _ = corpus_files
    args = ["summary", "--tsv", "--no-sampling", "--no-filtering"] + (["--ignore", ignore] if ignore else []) + [bam]
    text = subprocess.run([oracle_exe] + args, capture_output=True, text=True, check=True).stdout
    assert check_summary(text, corpus, ignore) >= 200
