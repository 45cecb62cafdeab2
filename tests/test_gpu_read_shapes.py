"""Reads of exact shapes through the product, byte for byte against the CPU oracle: every CIGAR op (N, H, P, =, X next to D
and I, at the 32-op batch edge), long CIGARs in CG:B,I, IUPAC bases, N+ lists, SEQ * and unmapped-but-placed records, and
reads on both sides of every kernel capacity limit (read from the CUDA sources). Each case runs the default kernels, the
fused (MKP_FUSED=1) and tile (MKP_TILE=1) kernels with a motif so their focus bitmaps engage, and, where the records differ
on the ingest side, --host-ingest; CIGAR cases also run pileup-hemi, admission cases summary and sample-probs. The declared
limits (MM lists, codes, states) must fail with their message and no bedMethyl rows."""
import os
import random
import re
import subprocess
import sys

import pytest

from conftest import ROOT, run_oracle, run_product, same_text
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)
from test_read_shapes_cpu import Genome, kernel_constant, long_cigar_ops

import bamio

pytestmark = pytest.mark.gpu

KERNELS = [None, "MKP_FUSED", "MKP_TILE"]
DUPLEX = ("C+h?", "C+m?", "G-m?")
SPLICED = ("C+hmf?", "G-m?")     # spliced reads carry a code (f) the background lacks: coverage wrongly run across an N adds rows


def ceil16(x):
    return (x + 15) // 16 * 16


def span_with(g, contig, pos, base, k):
    """Length n of the exact-copy alignment at pos whose read holds exactly k of `base` (the last base of the span is one)."""
    ref, seen = g.contigs[contig], 0
    for n in range(len(ref) - pos):
        seen += ref[pos + n] == base
        if seen == k:
            return n + 1
    raise ValueError("contig too short")


def explicit(header, deltas, seed):
    """heads callable for Genome.add: one list whose calls follow the given deltas over the read's bases of its base."""
    def f(read):
        base = header[0]
        occ = [q for q, c in enumerate(read) if c == base]
        rng, out, k = random.Random(seed), [], -1
        for d in deltas:
            k += d + 1
            out.append((occ[k], rng.randrange(256)))
        return [(header, out)]
    return f


def mm_deltas(lead, total):
    """Deltas whose MM text `C+m?` + deltas + `;` is exactly total bytes: the lead deltas, then 2-digit deltas between 0s."""
    text = lambda ds: 5 + sum(1 + len(str(d)) for d in ds)
    ds = list(lead)
    while text(ds) + 5 <= total - 4:
        ds += [12, 0]
    while text(ds) < total - 2:
        ds.append(0)
    if text(ds) == total - 2:
        ds.append(0)
    elif text(ds) == total - 1:
        ds[-1] = 10                                     # one byte longer
    assert text(ds) == total, (text(ds), total)
    return ds


# ---------------------------------------------------------------------------------------------------------------------------
# case builders: Genome -> (genome, options)

def case_cigar_ops():
    g = Genome(101, c1=30000)
    g.background("c1", 0, 30000, heads=DUPLEX)
    ref = g.contigs["c1"]
    batch31 = [("M" if k % 2 == 0 else "ID"[k % 4 == 1], 6 if k % 2 == 0 else 1) for k in range(31)]
    shapes = [
        (1000, [("S", 5), ("M", 300), ("N", 800), ("M", 250), ("S", 3)]),
        (3000, [("M", 40), ("N", 50), ("M", 30), ("N", 60), ("I", 2), ("M", 20), ("N", 0), ("M", 25), ("D", 3), ("N", 40),
                ("M", 30), ("N", 100), ("M", 50)]),
        (4500, batch31 + [("N", 200), ("M", 100)]),                    # N as op 31, the last of the first 32-op batch
        (5500, batch31 + [("M", 4), ("N", 200), ("M", 100)]),          # N as op 32, the first of the second
        (6500, [("M", 30), ("N", 0), ("M", 30), ("N", 0), ("N", 120), ("M", 40)]),
        (8000, [("M", 100), ("D", 5), ("N", 300), ("I", 4), ("M", 80), ("I", 3), ("N", 200), ("D", 2), ("M", 90)]),
        (11000, [("H", 20), ("S", 5), ("M", 150), ("P", 4), ("M", 60), ("I", 2), ("P", 1), ("D", 3), ("M", 80), ("H", 15)]),
        (13000, [("=", 50), ("X", 2), ("=", 30), ("N", 200), ("X", 1), ("=", 20), ("D", 3), ("I", 2), ("=", 40), ("X", 3),
                 ("M", 30), ("N", 0), ("P", 2), ("=", 25), ("H", 4)]),
        (15000, [("S", 10), ("D", 4), ("M", 200)]),
        (15500, [("S", 10), ("I", 5), ("M", 200)]),
        (16000, [("D", 3), ("M", 120), ("I", 2)]),
        (16500, [("H", 3), ("I", 3), ("X", 1), ("M", 120)]),
    ]
    for pos, cig in shapes:
        g.add_both("c1", pos, cig, heads=SPLICED if any(op == "N" and n for op, n in cig) else DUPLEX)
    # CpGs split by a junction or a deletion: C aligned and G skipped, C deleted and G aligned
    c = ref.index("CG", 18000)
    g.add_both("c1", c - 150, [("M", 151), ("N", 150), ("M", 100)], heads=SPLICED)
    c = ref.index("CG", c + 400)
    g.add_both("c1", c - 150, [("M", 151), ("D", 6), ("M", 100)], heads=DUPLEX)
    c = ref.index("CG", c + 400)
    g.add_both("c1", c - 150, [("M", 150), ("D", 1), ("M", 100)], heads=DUPLEX)
    c = ref.index("CG", c + 400)
    g.add_both("c1", c - 150, [("M", 150), ("N", 1), ("M", 100)], heads=SPLICED)
    # calls on the last aligned base: a forward read ending on a CpG's C, a reverse one ending on its G
    c = ref.index("CG", c + 400)
    g.add("c1", c - 300, [("S", 4), ("=", 301), ("S", 6)], heads=DUPLEX, frac=1.0)
    g.add("c1", c - 299, [("=", 301)], rev=True, heads=DUPLEX, frac=1.0)
    return g, dict(hemi=True)


def case_long_cigar_forms():
    g = Genome(102, c1=40000)
    g.background("c1", 0, 40000, heads=DUPLEX)
    for k, (pos, at) in enumerate(((3000, "first"), (9000, "middle"), (15000, "last"), (22000, "last"))):
        g.add_both("c1", pos, long_cigar_ops(3000, k), heads=DUPLEX, long_cigar=True, cg_at=at)
    return g, dict(hemi=True, host=True, region="c1:5000-17000")


def case_ncigar_caps():
    g = Genome(103, c1=50000, tl0=20000, tl1=20000)
    g.background("c1", 0, 50000, depth=6)
    cq, tl = kernel_constant("MKP_CQ_CAP"), kernel_constant("TL_MAXCIG")
    for k, n in enumerate((cq - 1, cq, cq + 1)):
        g.add_both("c1", 2000 + 14000 * k, long_cigar_ops(n, n), copies=1)
    # TL_MAXCIG: without N (a reference skip sends a read to the generic kernels), first in its chunk, and padded so that the
    # two reads fill the first tile window alone: the tile kernel keeps the read at the limit from start to finish (no other
    # read takes arena room before it) and refuses the one past it
    blk = ceil16(kernel_constant("MKP_TL_WIN") // 2 + 1)
    for contig, n in (("tl0", tl), ("tl1", tl + 1)):
        ops = long_cigar_ops(n - 1, n, cyc="M=IXDMPX=M") + [("S", 1)]
        for rev in (False, True):
            g.add(contig, 40, ops, rev=rev, heads=("C+m?",), block=blk)
        g.background(contig, 0, 20000, depth=6, min_pos=41)
    return g, dict(host=True)


def case_query_length_16k():
    g = Genome(104, c1=60000)
    g.background("c1", 0, 60000, depth=6)
    cum = kernel_constant("CUM_CAP") * 32
    for k, n in enumerate((cum, cum + 1)):
        g.add_both("c1", 3000 + 25000 * k, [("S", 10), ("M", n - 40), ("I", 5), ("M", 25)], copies=1)
    return g, {}


def case_query_length_64k():
    g = Genome(105, c1=220000)
    g.background("c1", 0, 220000, depth=4, mean_len=3000)
    for k, n in enumerate((65535, 65536, 65537)):
        g.add_both("c1", 2000 + 70000 * k, [("S", 3), ("M", n - 20), ("D", 2), ("M", 12), ("S", 5)], copies=1)
    return g, {}


def case_fused_block():
    g = Genome(106, c1=120000)
    g.background("c1", 0, 120000, depth=4, mean_len=3000)
    blk = kernel_constant("MKP_FZ_MAXBLK")
    for k, b in enumerate((blk - 1, blk, blk + 1)):
        for rev in (False, True):
            g.add("c1", 3000 + 36000 * k, [("S", 5), ("M", 15000), ("I", 2), ("M", 600), ("S", 1)], rev=rev, block=b)
    return g, {}


def case_entry_caps():
    g = Genome(107, c1=100000)
    g.background("c1", 0, 100000, depth=6)
    pos = 2000
    for cap in (kernel_constant("MKP_FZ_PCAP"), kernel_constant("TL_MAXENT")):
        for k in (cap, cap + 1):
            for rev in (False, True):
                n = span_with(g, "c1", pos, "G" if rev else "C", k)
                g.add("c1", pos, [("=", n)], rev=rev, heads=("C+m?",), frac=1.0)
            pos += n + 3000
    return g, {}


def case_tile_reads():
    win, nr = kernel_constant("MKP_TL_WIN"), kernel_constant("MKP_TL_READS")
    g = Genome(108, t12=20000, t13=20000)
    for contig, n in (("t12", nr), ("t13", nr + 1)):
        b = ceil16(-(-win // n))                       # n blocks start inside the first window of the chunk, the next one after it
        assert (n - 1) * b < win <= n * b
        for k in range(n):
            g.add(contig, 40, [("S", 3), ("M", 1200), ("S", 1)], rev=bool(k & 1), block=b)
        g.background(contig, 0, 20000, depth=8, min_pos=41)
    return g, {}


def case_mm_text():
    g = Genome(109, c1=60000)
    g.background("c1", 0, 60000, depth=6)
    pos = 1000
    for total in (1023, 1024, 1025):
        for rev in (False, True):
            ds = mm_deltas([], total)
            n = span_with(g, "c1", pos, "G" if rev else "C", sum(d + 1 for d in ds) + 3)
            rec = g.add("c1", pos, [("=", n)], rev=rev, heads=explicit("C+m?", ds, total))
            assert len(bamio.get_aux(rec, b"MM")) == total
        pos += n + 500
    # a two-digit delta across every byte offset of the parser's 128-byte window (leads of 2k or 3 + 2k bytes)
    for k in range(128):
        ds = mm_deltas([10] * (k & 1) + [0] * (k >> 1), 300)
        n = span_with(g, "c1", 20000 + 200 * k, "C", sum(d + 1 for d in ds) + 3)
        g.add("c1", 20000 + 200 * k, [("=", n)], heads=explicit("C+m?", ds, k))
    return g, {}


def case_iupac_and_n_lists():
    g = Genome(110, c1=30000)
    g.background("c1", 0, 30000)
    ref = g.contigs["c1"]
    for k, heads in enumerate((("C+m?",), ("N+a?",), ("C+m?", "N+a?"), ("C+h?", "C+m?", "N+a?"))):
        pos = 1000 + 6000 * k
        cig = [("S", 4), ("M", 900), ("N", 300), ("M", 400), ("I", 3), ("M", 300)]
        s = g.read_bases("c1", pos, cig)
        cs = [q for q, c in enumerate(s) if c in "CG"]
        subst = [(q, "NRY"[j % 3]) for j, q in enumerate(cs[::9])] + [(q, "N") for q in range(7, len(s), 61)]
        g.add_both("c1", pos, cig, seq=s, heads=heads, subst=subst)
    return g, dict(motif=["--cpg"], extra_motif=["--motif", "A", "0", "--motif", "CG", "0"])


def lists_heads(codes):
    """One single-code list per (base, code); codes are letters or numeric (ChEBI) codes."""
    return tuple("%s+%s?" % (b, c) for b, cs in codes for c in (cs if isinstance(cs, (list, tuple)) else list(cs)))


def chebi(n0, n):
    return [str(n0 + k) for k in range(n)]


def case_lists_and_codes():
    g = Genome(111, c1=30000)
    g.background("c1", 0, 30000)
    sixteen = lists_heads((("A", "abde"), ("C", "hmfc"), ("G", "gkno"), ("T", "tuvw")))
    assert len(sixteen) == kernel_constant("MAX_LISTS")
    g.add_both("c1", 2000, [("S", 3), ("M", 1200), ("D", 2), ("M", 800)], heads=sixteen)
    g.add_both("c1", 8000, [("S", 3), ("M", 1200), ("N", 200), ("M", 800)], heads=("C+hmfc?",))
    g.add_both("c1", 14000, [("M", 1500)], heads=("C+hm?", "G-hm?", "A+a?"))
    return g, {}


def case_admission():
    g = Genome(112, c1=20000)
    g.background("c1", 0, 20000)
    for k in range(10):
        if k % 5 == 2:                                  # primary with SEQ * (still counted by the pileup's depth buffer)
            g.add("c1", 8000, [("M", 700)], seq="", heads=None, mm_extra="", aux=(bamio.aux_z("MM", "C+m?;"), bamio.aux_b("ML", "C", [])))
        elif k % 5 == 4:                                # unmapped but placed, with calls
            g.add("c1", 8000, [], seq="".join(g.rng.choice("ACGT") for _ in range(600)), flag=4)
        else:
            g.add("c1", 8000, [("S", 2), ("M", 700 + 10 * k)], rev=bool(k & 1))
    g.add("c1", 12000, [], seq="".join(g.rng.choice("ACGT") for _ in range(900)), flag=4, rev=True)
    return g, dict(host=True, reports=True, depth=["--max-depth", "6"])


CASES = [
    ("cigar_ops", case_cigar_ops),
    ("long_cigar_forms", case_long_cigar_forms),
    ("ncigar_caps", case_ncigar_caps),
    ("query_length_16k", case_query_length_16k),
    ("query_length_64k", case_query_length_64k),
    ("fused_block", case_fused_block),
    ("entry_caps", case_entry_caps),
    ("tile_reads", case_tile_reads),
    ("mm_text", case_mm_text),
    ("iupac_and_n_lists", case_iupac_and_n_lists),
    ("lists_and_codes", case_lists_and_codes),
    ("admission", case_admission),
]


def product_with(kernel, flags, bam, out):
    if kernel:
        os.environ[kernel] = "1"
    try:
        return run_product(flags, bam, out)
    finally:
        os.environ.pop(kernel or "", None)


def check_pileup(oracle_exe, flags, bam, tmp_path, kernels, min_rows, oracle_flags=None):
    exp = run_oracle(oracle_exe, oracle_flags or flags, bam, str(tmp_path / "o.bed"))
    assert exp.count("\n") > min_rows, "degenerate test input"
    for kernel in kernels:
        rc, got = product_with(kernel, flags, bam, str(tmp_path / "g.bed"))
        assert rc == 0, (kernel, flags)
        assert same_text(got, exp), (kernel, flags)


@pytest.mark.parametrize("name,build", CASES, ids=[c[0] for c in CASES])
def test_read_shapes_match_oracle(name, build, native_lib, oracle_exe, hemi_oracle_exe, tmp_path):
    g, opt = build()
    bam, fa = g.write(tmp_path)
    motif = opt.get("motif", ["--cpg"])
    base = ["--ref", fa, "--no-filtering"] + opt.get("depth", [])
    check_pileup(oracle_exe, motif + base, bam, tmp_path, KERNELS, 200)
    if "extra_motif" in opt:
        check_pileup(oracle_exe, opt["extra_motif"] + base, bam, tmp_path, KERNELS, 200)
    # every position, estimated thresholds, interval 7001: the default kernels
    check_pileup(oracle_exe, ["-i", "7001"] + opt.get("depth", []), bam, tmp_path, [None], 500)
    if opt.get("host"):
        check_pileup(oracle_exe, motif + base + ["--host-ingest"], bam, tmp_path, [None], 200, oracle_flags=motif + base)
    if "region" in opt:
        flags = ["--region", opt["region"], "--cpg"] + base
        check_pileup(oracle_exe, flags, bam, tmp_path, KERNELS, 100)
        check_pileup(oracle_exe, flags + ["--host-ingest"], bam, tmp_path, [None], 100, oracle_flags=flags)
    if opt.get("hemi"):
        from test_gpu_hemi import run_hemi, run_oracle_hemi
        args = [bam, "-r", fa, "--cpg", "--no-filtering"]
        exp = run_oracle_hemi(hemi_oracle_exe, args, str(tmp_path / "oh.bed"))
        assert exp.count("\n") > 200
        for extra in ([], ["--host-ingest"]):
            rc, got = run_hemi(args + extra, str(tmp_path / "gh.bed"))
            assert rc == 0 and same_text(got, exp)
    if opt.get("reports"):
        from test_gpu_summary import oracle, product
        for cmd, args in (("summary", ["--tsv", "--no-sampling"]), ("summary", ["--tsv", "--no-sampling", "--only-mapped"]),
                          ("sample-probs", ["--no-sampling"])):
            exp = oracle(oracle_exe, cmd, args + [bam])
            assert exp.count("\n") > 3
            assert product(cmd, args + [bam], tmp_path) == exp, (cmd, args)


def test_cg_65536_ops_equals_65535_in_the_core(native_lib, oracle_exe, tmp_path):
    """The most ops the core can hold, and one more in CG:B,I (the last op split in two): same bases, same rows."""
    cig = long_cigar_ops(65535, 7)
    assert cig[-1] == ("M", 5)
    outs = []
    for k, (ops, long_cigar) in enumerate(((cig, False), (cig[:-1] + [("M", 2), ("M", 3)], True))):
        g = Genome(113, c1=150000)
        g.background("c1", 0, 150000, depth=4, mean_len=3000)
        g.add_both("c1", 5000, ops, copies=1, long_cigar=long_cigar)
        d = tmp_path / str(k)
        d.mkdir()
        bam, fa = g.write(d)
        flags = ["--cpg", "--ref", fa, "--no-filtering"]
        check_pileup(oracle_exe, flags, bam, d, KERNELS, 1000)
        check_pileup(oracle_exe, flags + ["--host-ingest"], bam, d, [None], 1000, oracle_flags=flags)
        check_pileup(oracle_exe, flags + ["--region", "c1:40000-120000"], bam, d, [None], 1000)
        outs.append(open(d / "o.bed").read())
    assert outs[0] == outs[1]


# ---------------------------------------------------------------------------------------------------------------------------
# declared limits: an error, never a wrong answer

def n_states(records):
    """Distinct (base, mod code) pairs named by the MM lists of the records."""
    out = set()
    for r in records:
        for head in bamio.get_aux(r, b"MM").decode().split(";")[:-1]:
            m = re.match(r"([ACGTUN])[+-](\d+|[a-z]+)", head)
            codes = [m.group(2)] if m.group(2).isdigit() else list(m.group(2))
            out |= {(m.group(1), c) for c in codes}
    return len(out)


LIMITS = [
    ("lists_17", [lists_heads((("A", "abde"), ("C", "hmfc"), ("G", "gkno"), ("T", "tuvw"))) + ("C-z?",)], "more than 16 MM lists in one read"),
    ("codes_5_in_a_list", [("C+hmfcz?",)], "more than 4 codes in one MM list"),
    ("codes_8_at_a_position", [("C+hmfc?", "C+abde?")], "7 at one position"),
    ("states_33", [lists_heads((("A", "abde"), ("C", "hmfc"), ("G", "gkno"), ("T", "tuvw"))),
                   lists_heads((("A", chebi(1000, 4)), ("C", chebi(2000, 4)), ("G", chebi(3000, 4)), ("T", chebi(4000, 4)))),
                   lists_heads((("A", chebi(1100, 1)),))], "more than 32 distinct (base, mod code) states"),
]


@pytest.mark.parametrize("name,reads,msg", LIMITS, ids=[c[0] for c in LIMITS])
def test_declared_limits_fail_without_rows(name, reads, msg, native_lib, tmp_path):
    g = Genome(114, c1=20000)
    g.background("c1", 0, 20000, heads=("C+m?",))
    for k, heads in enumerate(reads):
        g.add("c1", 6000 + 100 * k, [("M", 1500)], heads=heads, frac=0.5)
    if name == "states_33":
        assert n_states(g.records) == kernel_constant("MAX_STATES") + 1
    bam, fa = g.write(tmp_path)
    for kernel in KERNELS:
        out = tmp_path / ("g%s.bed" % kernel)
        env = dict(os.environ, **({kernel: "1"} if kernel else {}))
        code = "import sys; sys.path.insert(0, %r); import modkit_b200; sys.exit(modkit_b200.pileup_main(sys.argv[1:]))" % ROOT
        p = subprocess.run([sys.executable, "-c", code, "--cpg", "--ref", fa, "--no-filtering", "--quiet", bam, str(out)],
                           capture_output=True, text=True, env=env)
        assert p.returncode == 1 and msg in p.stderr, (kernel, p.returncode, p.stderr[-400:])
        assert not out.exists() or out.stat().st_size == 0, kernel


def test_declared_limits_at_the_limit_match_oracle(native_lib, oracle_exe, tmp_path):
    """16 lists, 4 codes in a list, 7 codes at a position and 32 states are inside the limits: rows equal the oracle's."""
    g = Genome(115, c1=30000)
    g.background("c1", 0, 30000, heads=("C+m?",))
    g.add("c1", 3000, [("M", 1500)], heads=lists_heads((("A", "abde"), ("C", "hmfc"), ("G", "gkno"), ("T", "tuvw"))), frac=0.5)
    g.add("c1", 9000, [("M", 1500)], heads=("C+hmfc?", "C+abd?"), frac=0.5)
    g.add("c1", 15000, [("M", 1500)], heads=lists_heads((("A", chebi(1000, 4)), ("C", chebi(2000, 4)), ("G", chebi(3000, 4)),
                                                         ("T", chebi(4000, 1)))), frac=0.5)
    assert n_states(g.records) == kernel_constant("MAX_STATES")
    bam, fa = g.write(tmp_path)
    check_pileup(oracle_exe, ["--ref", fa, "--no-filtering", "--motif", "C", "0", "--motif", "A", "0"], bam, tmp_path, KERNELS, 500)
    check_pileup(oracle_exe, ["--no-filtering"], bam, tmp_path, [None], 500)


def test_chunk_without_reads_runs_only_rank_and_row_kernels(native_lib):
    """A chunk without reads through every pass: no rows, and mkp_kernel_launches counts the kernels issued, which are the
    rank and row kernels only. Decode, counting and emit kernels have nothing to do and are not launched."""
    import numpy as np
    import modkit_b200
    ctx = modkit_b200.Context(0)
    ctx.set_params(modkit_b200.make_params())
    end = 100000
    focus = np.zeros((end + 31) // 32, dtype=np.uint32)
    focus[::7] = 0x01010101
    for with_focus in (False, True):
        ch = modkit_b200.Chunk()
        ch.start, ch.end = 0, end
        if with_focus:
            ch.focus_pos = ch.focus_neg = focus.ctypes.data
        l0 = ctx.kernel_launches
        ctx._check(ctx._lib.mkp_upload_chunk(ctx._h, ch))
        # with focus bitmaps the upload ranks them (3 kernels), builds the word records (1) and the tile table (1)
        assert ctx.kernel_launches - l0 == (5 if with_focus else 0)
        l0 = ctx.kernel_launches
        st = ctx.pileup_resident()
        assert st.n_rows == 0 and st.n_calls == 0 and len(ctx.fetch_rows()) == 0
        # hot-mark pass: rank of the marks (3) and word records (1); focus-rank pass: no rank; both: row count and scan (4),
        # and the focus-rank pass emits without reading the row count back (1)
        assert ctx.kernel_launches - l0 == (5 if with_focus else 8)
        l0 = ctx.kernel_launches
        hist, _, _ = ctx.sample_histogram()
        assert not hist.any() and ctx.kernel_launches == l0
    l0 = ctx.kernel_launches
    st = ctx.hemi_resident([0], 1)
    assert st.n_rows == 0 and len(ctx.fetch_hemi_rows()) == 0
    assert ctx.kernel_launches - l0 == 7            # rank of focus_pos (3), row count and scan (4)
