"""Reads shaped for k_parse's streaming select, byte for byte against the CPU oracle: SEQ lengths on both sides of the 32-base
block and the 1024-base round, odd lengths, every 16-byte alignment of the SEQ, more tokens in one round than one 32-token
window holds, token counts at the window edges, tokens only in the last partial round, two lists of one base with different
deltas (no alias), aliased lists at shifted text offsets, lists on two bases, N and '.' lists, a token one past the last
occurrence (the read is skipped), and a 200 kb read with about 3 000 tokens per list. Every case runs the default kernels with
--cpg and over all positions, pileup-hemi, and summary / sample-probs, which decode through the same k_parse."""
import random

import pytest

from conftest import same_text
from test_gpu_read_shapes import check_pileup
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)
from test_read_shapes_cpu import Genome

import bamio

pytestmark = pytest.mark.gpu

DUPLEX = ("C+h?", "C+m?", "G-m?")   # background lists: calls on both strands, so pileup-hemi has rows


def picked(spec, seed):
    """heads callable for Genome.add: spec = [(header, pick)], pick(n_occ) -> occurrence indices of the list's base (read
    orientation) that carry a call. Probabilities stay below 85 so three lists at one position sum to at most 252."""
    def f(read):
        rng, out = random.Random(seed), []
        for header, pick in spec:
            occ = [q for q, c in enumerate(read) if header[0] == "N" or c == header[0]]
            out.append((header, [(occ[k], rng.randrange(85)) for k in sorted(set(pick(len(occ))))]))
        return out
    return f


def first(k):
    return lambda n: range(min(k, n))


def last(k):
    return lambda n: range(max(0, n - k), n)


def every(step, off=0):
    return lambda n: range(off, n, step)


def site(g, contig, start, base):
    """First position at or after start whose reference base is `base`."""
    return g.contigs[contig].index(base, start)


def case_lengths():
    g = Genome(201, c1=80000)
    g.background("c1", 0, 80000, depth=4, heads=DUPLEX)
    pos = 1000
    for n in (1, 2, 31, 32, 33, 63, 65, 777, 1023, 1024, 1025, 1057, 2049):
        for rev in (False, True):
            for hops in range(4):                       # 0-3 hard clips: 4 n_cigar bytes each shift the SEQ's 16-byte alignment
                p = site(g, "c1", pos, "G" if rev else "C") if n == 1 else pos
                cig = [("H", 1 + k) for k in range(hops)] + [("=", n)]
                g.add("c1", p, cig, rev=rev, heads=("C+h?", "C+m?"), frac=1.0)
                pos = p + 13
        pos += n + 200
    return g


def case_dense_tokens():
    g = Genome(202, c1=60000)
    ref = list(g.contigs["c1"])
    ref[5000:5600] = "C" * 600                          # a poly-C run: every base of several rounds is a token
    ref[9000:9800] = "CG" * 400
    g.contigs["c1"] = "".join(ref)
    g.background("c1", 0, 60000, depth=4, heads=DUPLEX)
    for rev in (False, True):
        g.add("c1", 4800, [("=", 1000)], rev=rev, frac=1.0)
        g.add("c1", 8900, [("=", 1500)], rev=rev, frac=1.0)
    pos = 14000
    for k in (1, 31, 32, 33, 63, 64, 65, 96, 97):      # window edges, tokens spread over the read and packed at its end
        for rev in (False, True):
            g.add("c1", pos, [("=", 3000)], rev=rev, heads=picked([("C+h?", first(k)), ("C+m?", first(k))], k))
            g.add("c1", pos + 500, [("=", 1100)], rev=rev, heads=picked([("C+m?", last(k))], k))
        pos += 3500
    return g


def case_lists():
    g = Genome(203, c1=40000)
    g.background("c1", 0, 40000, depth=4, heads=DUPLEX)
    pos = 1000
    shapes = [
        [("C+h?", every(3)), ("C+m?", every(2, 1))],                    # one base, different deltas: both windows live
        [("C+h?", every(2)), ("C+m?", every(5)), ("C+f?", first(70))],
        [("A+a?", every(4)), ("C+h?", every(2)), ("C+m?", every(2))],      # two needed bases, then an alias
        [("C+m?", every(3)), ("A+a?", every(5)), ("G-m?", every(7))],
        [("N+a?", every(11)), ("C+m?", every(2))],
        [("C+h.", every(2)), ("C+m.", every(2))],
        [("C+m.", every(3)), ("A+a?", every(9))],
    ]
    for j, spec in enumerate(shapes):
        for rev in (False, True):
            g.add("c1", pos, [("S", 3), ("M", 1800), ("I", 2), ("M", 700)], rev=rev, heads=picked(spec, j))
        pos += 2800
    # aliased lists whose delta texts start at every byte offset mod 4 (and mod 16): a leading list of 1-8 tokens
    for k in range(1, 9):
        for rev in (False, True):
            g.add("c1", pos, [("=", 1500)], rev=rev, heads=picked([("A+a?", first(k)), ("C+h?", every(2)), ("C+m?", every(2))], k))
        pos += 1600
    return g


def case_past_last():
    g = Genome(204, c1=20000)
    g.background("c1", 0, 20000, depth=6, heads=DUPLEX)
    for k, (n, rev) in enumerate(((700, False), (700, True), (1024, False), (1025, True))):
        for extra in (0, 1):                            # the token on the last occurrence, and one past it (the read errors)
            pos = 3000 + 3000 * k + 100 * extra
            s = g.read_bases("c1", pos, [("=", n)])
            read = bamio.revcomp(s) if rev else s
            mm = "C+m?,%d;" % (read.count("C") - 1 + extra)
            g.add("c1", pos, [("=", n)], rev=rev, seq=s, heads=None,
                  aux=(bamio.aux_z("MM", mm), bamio.aux_b("ML", "C", [230])))
    return g


def case_long_read():
    g = Genome(205, c1=230000)
    g.background("c1", 0, 230000, depth=3, mean_len=3000, heads=DUPLEX)
    for rev in (False, True):
        g.add("c1", 10000 + 1000 * rev, [("S", 7), ("M", 120000), ("D", 3), ("M", 80000), ("S", 5)], rev=rev, frac=0.06)
    return g


CASES = [
    ("lengths", case_lengths),
    ("dense_tokens", case_dense_tokens),
    ("lists", case_lists),
    ("past_last", case_past_last),
    ("long_read", case_long_read),
]


@pytest.mark.parametrize("name,build", CASES, ids=[c[0] for c in CASES])
def test_select_shapes_match_oracle(name, build, native_lib, oracle_exe, hemi_oracle_exe, tmp_path):
    g = build()
    bam, fa = g.write(tmp_path)
    check_pileup(oracle_exe, ["--cpg", "--ref", fa, "--no-filtering"], bam, tmp_path, [None], 200)
    check_pileup(oracle_exe, ["--no-filtering"], bam, tmp_path, [None], 500)
    from test_gpu_hemi import run_hemi, run_oracle_hemi
    args = [bam, "-r", fa, "--cpg", "--no-filtering"]
    exp = run_oracle_hemi(hemi_oracle_exe, args, str(tmp_path / "oh.bed"))
    assert exp.count("\n") > 100
    rc, got = run_hemi(args, str(tmp_path / "gh.bed"))
    assert rc == 0 and same_text(got, exp)
    from test_gpu_summary import oracle, product
    for cmd, extra in (("summary", ["--tsv", "--no-sampling"]), ("sample-probs", ["--no-sampling"])):
        exp = oracle(oracle_exe, cmd, extra + [bam])
        assert exp.count("\n") > 3
        assert product(cmd, extra + [bam], tmp_path) == exp, (cmd, extra)
