"""Reads of exact shapes, built record by record with tools/bamio.py (make_record, mm_for): every CIGAR op, long CIGARs stored
in CG:B,I, IUPAC bases, reads at the kernels' capacity limits. This file holds the builder the GPU suite
(test_gpu_read_shapes.py) shares and the CPU checks: the builder round-trips every shape, and a long CIGAR gives the same
oracle output (pileup, pileup-hemi, summary) and the same packed chunk whether it sits in the core or in CG:B,I."""
import ctypes
import os
import random
import re
import subprocess

import pytest

from conftest import ROOT, run_oracle
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)

import bamio

CSRC = os.path.join(ROOT, "modkit_b200", "csrc")


def kernel_constant(name):
    """A capacity constant of the CUDA sources (`#define NAME expr` or `NAME = expr` in a constexpr), read at test time so the
    boundary reads follow a retune."""
    text = "".join(open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".cu")))
    m = re.search(r"#define\s+%s\s+([^\n]+)" % name, text) or re.search(r"\b%s\s*=\s*([^,;]+)[,;]" % name, text)
    assert m, name
    expr = m.group(1).split("//")[0].strip()
    expr = re.sub(r"\b(MKP_[A-Z_]+)\b", lambda k: str(kernel_constant(k.group(1))), expr)
    assert re.fullmatch(r"[\d\s*()+-]+", expr), (name, expr)
    return int(eval(expr))


def block_bytes(rec):
    """Bytes of a record's block in a packed chunk: CIGAR, packed SEQ, ML, MM (before the 16-byte alignment)."""
    f = bamio.rec_fields(rec)
    mm, ml = bamio.get_aux(rec, b"MM"), bamio.get_aux(rec, b"ML")
    return 4 * len(full_cigar(rec)) + (f["l_seq"] + 1) // 2 + (len(mm) + len(ml) if mm is not None and ml is not None else 0)


def full_cigar(rec):
    """[(op, len)] of a record, the CG:B,I array when the core holds its placeholder (the rule of the product's packer)."""
    f = bamio.rec_fields(rec)
    words = f["cigar"]
    cg = bamio.get_aux(rec, b"CG")
    if len(words) == 2 and words[0] & 15 == 4 and words[0] >> 4 == f["l_seq"] and cg is not None:
        words = list(memoryview(cg).cast("I"))
    return [(bamio.CIGAR_OPS[w & 15], w >> 4) for w in words]


def seq_text(rec):
    f = bamio.rec_fields(rec)
    return "".join(bamio.SEQ_NIB[(f["seq"][i >> 1] >> (0 if i & 1 else 4)) & 15] for i in range(f["l_seq"]))


class Genome:
    """One or more random contigs and the records placed on them. Shaped reads go through add(); background() lays ordinary
    reads (M with a few I/D, both strands, calls on most C) over a range so rows exist around and under the shaped reads."""

    def __init__(self, seed, **contigs):
        self.rng = random.Random(seed)
        self.contigs = {name: "".join(self.rng.choice("ACGT") for _ in range(n)) for name, n in contigs.items()}
        self.names = list(self.contigs)
        self.records = []
        self.n = 0

    def read_bases(self, contig, pos, cigar):
        """Stored SEQ of a read aligned at pos with this CIGAR: M copies the reference with a few mismatches, = copies it,
        X differs from it, I and S are random, D N H P add no base."""
        ref, rng, out, r = self.contigs[contig], self.rng, [], pos
        for op, n in cigar:
            if op in "M=X":
                for k in range(n):
                    b = ref[r + k]
                    if op == "X" or (op == "M" and rng.random() < 0.03):
                        b = rng.choice([c for c in "ACGT" if c != b])
                    out.append(b)
            elif op in "IS":
                out.append("".join(rng.choice("ACGT") for _ in range(n)))
            if op in "MDN=X":
                r += n
        return "".join(out)

    def calls(self, read, heads, frac):
        """[(header, calls)] for mm_for: lists of one base share their positions, and their probabilities sum to <= 255."""
        by_base = {}
        for h in heads:
            by_base.setdefault(h[0], []).append(h)
        out = {}
        for base, hs in by_base.items():
            codes = [len(re.match(r".[+-]([a-z]+|\d+)", h).group(1)) if not h[2:-1].isdigit() else 1 for h in hs]
            picks = [q for q, c in enumerate(read) if (base == "N" or c == base) and self.rng.random() < frac]
            lists = {h: [] for h in hs}
            for q in picks:
                cut = sorted(self.rng.randrange(256) for _ in range(sum(codes)))
                ps = [cut[0]] + [b - a for a, b in zip(cut, cut[1:])]
                k = 0
                for h, nc in zip(hs, codes):
                    lists[h].append((q, tuple(ps[k:k + nc]) if nc > 1 else ps[k]))
                    k += nc
            out.update(lists)
        return [(h, out[h]) for h in heads]

    def add(self, contig, pos, cigar, rev=False, heads=("C+h?", "C+m?"), frac=0.8, subst=(), flag=0, seq=None, block=None,
            mm_extra="", **kw):
        """One record; returns it. subst: [(query index, letter)] applied to the stored SEQ (IUPAC letters); block: pad the read
        with trailing soft-clipped A (no calls: the lists are on C/G) until its packed block has exactly this many bytes;
        mm_extra: MM text appended after the generated lists (lists without calls); heads=None writes no MM/ML, a callable
        heads(read) returns the [(header, calls)] of the read (read orientation) itself."""
        s = self.read_bases(contig, pos, cigar) if seq is None else seq
        for q, c in subst:
            s = s[:q] + c + s[q + 1:]
        assert block is None or cigar[-1][0] == "S", "a padded read ends with a soft clip"
        cig = list(cigar)
        while True:
            read = bamio.revcomp(s) if rev else s
            state = self.rng.getstate()
            if callable(heads):                             # explicit [(header, calls)] of the read-orientation bases
                mm, ml = bamio.mm_for(s, rev, heads(read))
            else:
                mm, ml = bamio.mm_for(s, rev, self.calls(read, heads, frac)) if heads is not None else (None, None)
            if mm is not None:
                mm += mm_extra
            self.n += 1
            rec = bamio.make_record(self.names.index(contig), pos, flag | (16 if rev else 0), cig, s, mm, ml, name="s%d" % self.n, **kw)
            if block is None or block_bytes(rec) >= block:
                break
            self.rng.setstate(state)                        # the same calls on the longer read
            self.n -= 1
            s += "A" * max(1, 2 * (block - block_bytes(rec)) - 1)
            cig = cigar[:-1] + [("S", cigar[-1][1] + len(s) - bamio.cigar_spans(cigar)[0])]
        assert block is None or block_bytes(rec) == block, (block_bytes(rec), block)
        self.records.append(rec)
        return rec

    def add_both(self, contig, pos, cigar, copies=2, **kw):
        """copies forward and copies reverse records of one shape (the same bases, independent calls)."""
        s = self.read_bases(contig, pos, cigar) if kw.get("seq") is None else kw.pop("seq")
        return [self.add(contig, pos, cigar, rev=bool(k & 1), seq=s, **kw) for k in range(2 * copies)]

    def background(self, contig, lo, hi, depth=10, mean_len=1500, heads=("C+h?", "C+m?"), min_pos=0):
        """Reads starting in [lo - len / 2, hi), never before min_pos."""
        L = len(self.contigs[contig])
        n = depth * (hi - lo) // mean_len
        for _ in range(n):
            ln = self.rng.randint(mean_len // 2, mean_len * 3 // 2)
            pos = self.rng.randrange(max(min_pos, lo - ln // 2), max(min_pos + 1, min(L - ln - 10, hi)))
            cig, left = [("S", self.rng.randint(0, 20))], ln
            while left > 0:
                m = min(left, self.rng.randint(50, 400))
                cig.append(("M", m))
                left -= m
                if left > 0:
                    cig.append((self.rng.choice("ID"), self.rng.randint(1, 4)))
            cig = [c for c in cig if c[1]]
            if bamio.cigar_spans(cig)[1] + pos > L:
                continue
            self.add(contig, pos, cig, rev=self.rng.random() < 0.5, heads=heads)

    def write(self, dirpath, name="shapes"):
        bam = os.path.join(str(dirpath), name + ".bam")
        fa = os.path.join(str(dirpath), name + ".fa")
        bamio.bam_of([(c, len(s)) for c, s in self.contigs.items()], self.records).write(bam, index=True)
        bamio.write_fasta(fa, self.contigs)
        return bam, fa


def long_cigar_ops(n_ops, seed, cyc="M=IXDMNX=MPM"):
    """A CIGAR of n_ops short ops between a soft clip and a final M, cycling through `cyc` (by default every op that consumes
    query or reference, M I D N = X, plus P)."""
    rng = random.Random(seed)
    ops = [("S", 7)]
    while len(ops) < n_ops - 1:
        op = cyc[len(ops) % len(cyc)]
        ops.append((op, rng.randint(1, 3) if op in "M=X" else 1))
    ops.append(("M", 5))
    return ops


# ---------------------------------------------------------------------------------------------------------------------------
# builder sanity

SHAPES = [
    ("N_mid", [("S", 4), ("M", 40), ("N", 300), ("M", 30)], "ACGT"),
    ("H_P", [("H", 9), ("M", 20), ("P", 3), ("M", 10), ("H", 2)], "ACGT"),
    ("eqx", [("=", 5), ("X", 2), ("D", 3), ("N", 0), ("I", 2), ("=", 10)], "ACGT"),
    ("soft_D", [("S", 3), ("D", 2), ("M", 20)], "ACGT"),
    ("soft_I", [("S", 3), ("I", 2), ("M", 20)], "ACGT"),
    ("iupac", [("M", 30)], "NRY"),
    ("long", long_cigar_ops(3000, 1), "ACGT"),
]


@pytest.mark.parametrize("long_cigar,cg_at", [(False, "last"), (True, "first"), (True, "middle"), (True, "last")])
@pytest.mark.parametrize("name,cigar,alphabet", SHAPES, ids=[s[0] for s in SHAPES])
def test_builder_round_trips(name, cigar, alphabet, long_cigar, cg_at):
    g = Genome(3, c1=20000)
    subst = [(k, random.Random(k).choice(alphabet)) for k in range(0, bamio.cigar_spans(cigar)[0], 7)]
    rec = g.add("c1", 500, cigar, rev=True, heads=("C+m?", "N+a?"), subst=subst, long_cigar=long_cigar, cg_at=cg_at)
    f = bamio.rec_fields(rec)
    assert full_cigar(rec) == cigar and f["pos"] == 500 and f["flag"] == 16 and f["qual"] == b"\xff" * f["l_seq"]
    s = seq_text(rec)
    assert len(s) == bamio.cigar_spans(cigar)[0] and all(s[q] == c for q, c in subst)
    beg, end = bamio.ref_span(f)
    assert (beg, end) == (500, 500 + bamio.cigar_spans(cigar)[1])
    assert f["cigar"][0] >> 4 == f["l_seq"] if long_cigar else len(f["cigar"]) == len(cigar)
    tags = [t for t, *_ in bamio.iter_aux(rec, f["aux_off"])]
    if long_cigar:
        assert tags == {"first": [b"CG", b"MM", b"ML"], "middle": [b"MM", b"CG", b"ML"], "last": [b"MM", b"ML", b"CG"]}[cg_at]
    # MM deltas: exact letters of the read orientation only (an IUPAC base is never a C); N lists count every base
    read = bamio.revcomp(s)
    mm = bamio.get_aux(rec, b"MM").decode()
    c_list, n_list = mm.split(";")[:2]
    occ_c = [q for q, c in enumerate(read) if c == "C"]
    got, k = [], -1
    for d in c_list.split(",")[1:]:
        k += int(d) + 1
        got.append(occ_c[k])
    assert all(read[q] == "C" for q in got)
    assert sum(1 for _ in n_list.split(",")[1:]) + len(got) == len(bamio.get_aux(rec, b"ML"))


def test_builder_seq_star_and_unmapped_placed():
    rec = bamio.make_record(0, 7, 0, [("M", 40)], "", "C+m?;", [])
    f = bamio.rec_fields(rec)
    assert f["l_seq"] == 0 and f["seq"] == b"" and f["qual"] == b"" and bamio.ref_span(f) == (7, 47)
    assert bamio.get_aux(rec, b"MM") == b"C+m?;" and bamio.get_aux(rec, b"ML") == b""
    rec = bamio.make_record(0, 9, 4, [], "ACGT", "C+m?,0;", [200])
    f = bamio.rec_fields(rec)
    assert f["cigar"] == [] and f["flag"] == 4 and seq_text(rec) == "ACGT" and bamio.ref_span(f) == (9, 10)


def shape_records(g):
    """Every SHAPES CIGAR in the core and in CG:B,I, plus a read consuming no reference and an unmapped-but-placed one."""
    recs = []
    for k, (name, cigar, _) in enumerate(SHAPES):
        for long_cigar in (False, True):
            recs.append(g.add("c1", 1000 + 3000 * k, cigar, rev=bool(k & 1), long_cigar=long_cigar))
    recs.append(g.add("c1", 30000, [("S", 5), ("I", 3), ("S", 2)]))
    recs.append(g.add("c1", 31000, [], seq="ACGTACGTAC", flag=4))
    return recs


def test_ref_span_matches_oracle_endpos(oracle_exe, tmp_path):
    """bamio.ref_span (the span the BAI writer indexes) is the oracle's endpos (htslib bam_endpos, CG:B,I applied), and the
    oracle sees the full CIGAR of a CG record."""
    g = Genome(4, c1=40000)
    recs = shape_records(g)
    bam, _ = g.write(tmp_path)
    got = {}
    for line in subprocess.run([oracle_exe, "endpos", bam], capture_output=True, text=True, check=True).stdout.splitlines():
        name, pos, end, n_cigar = line.split()
        got[name] = (int(pos), int(end), int(n_cigar))
    assert len(got) == len(recs)
    for rec in recs:
        f = bamio.rec_fields(rec)
        assert got[f["name"]] == bamio.ref_span(f) + (len(full_cigar(rec)),), f["name"]


def test_ref_span_matches_the_packers_fetch(tmp_path):
    """The record's reference end (bamio.ref_span, which the BAI writer uses) is the end the product's reader computes: a read
    overlaps [end - 1, end) and not [end, end + 1), for standard and CG:B,I CIGARs with N, D, P and H."""
    import modkit_b200
    g = Genome(4, c1=40000)
    spans = [bamio.ref_span(bamio.rec_fields(rec)) for rec in shape_records(g)]
    bam, _ = g.write(tmp_path)
    b = modkit_b200.Bam(bam, threads=1)
    for beg, end in spans:
        assert beg in b.pack(0, end - 1, end).headers()["ref_start"].tolist()
        assert beg not in b.pack(0, end, end + 1).headers()["ref_start"].tolist()


# ---------------------------------------------------------------------------------------------------------------------------
# long CIGARs: CG:B,I against the same CIGAR in the core

def long_cigar_pair(tmp_path, n_ops=3000, cg_at="last", seed=11):
    """Two BAMs with the same reads: ~n_ops-op CIGARs in the core, and the same CIGARs in CG:B,I (plus background reads)."""
    paths = []
    for long_cigar in (False, True):
        g = Genome(seed, c1=60000)
        g.background("c1", 0, 60000, depth=6, heads=("C+m?", "G-m?"))
        cig = long_cigar_ops(n_ops, seed)
        for k, pos in enumerate((2000, 9000, 21000)):
            g.add_both("c1", pos, cig, copies=2, heads=("C+m?", "G-m?"), long_cigar=long_cigar, cg_at=("first", "middle", "last")[k] if cg_at is None else cg_at)
        d = tmp_path / ("cg" if long_cigar else "std")
        d.mkdir()
        paths.append(g.write(d))
    return paths


@pytest.mark.parametrize("cg_at", ["first", "middle", "last"])
def test_oracle_long_cigar_equals_standard(cg_at, oracle_exe, hemi_oracle_exe, tmp_path):
    (std, fa), (cg, _) = long_cigar_pair(tmp_path, cg_at=cg_at)
    outs = []
    for bam in (std, cg):
        pile = run_oracle(oracle_exe, ["--no-filtering", "--cpg", "--ref", fa], bam, str(tmp_path / "o.bed"))
        allpos = run_oracle(oracle_exe, ["-i", "7000"], bam, str(tmp_path / "a.bed"))
        p = subprocess.run([hemi_oracle_exe, "pileup-hemi", "-t", "2", bam, "-r", fa, "--cpg", "--no-filtering", "-o", str(tmp_path / "h.bed")],
                           capture_output=True, text=True)
        assert p.returncode == 0, p.stderr
        summ = subprocess.run([oracle_exe, "summary", "--tsv", "--no-sampling", bam], capture_output=True, text=True, check=True).stdout
        outs.append((pile, allpos, open(tmp_path / "h.bed").read(), summ))
    assert outs[0] == outs[1]
    pile, allpos, hemi, summ = outs[0]
    assert pile.count("\n") > 1000 and allpos.count("\n") > 3000 and hemi.count("\n") > 500 and "C_pass_calls" in summ
    # the long reads contribute: the reads that span 9000-9100 are only the shaped ones and the background
    assert int(dict(ln.split("\t") for ln in summ.splitlines())["total_reads_used"]) > 12


def test_packer_long_cigar_equals_standard(tmp_path):
    import modkit_b200
    (std, _), (cg, _) = long_cigar_pair(tmp_path, cg_at=None)
    packs = []
    for bam in (std, cg):
        b = modkit_b200.Bam(bam, threads=2)
        pk = b.pack(0, 0, 60000)
        packs.append((pk.headers(), ctypes.string_at(pk.chunk().heap, pk.heap_bytes)))
    assert len(packs[0][0]) > 40 and max(packs[0][0]["n_cigar"]) >= 2999
    assert packs[0][0].tobytes() == packs[1][0].tobytes()
    assert packs[0][1] == packs[1][1]
