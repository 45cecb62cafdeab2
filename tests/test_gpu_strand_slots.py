"""Counter slots belong to a (position, reference strand) pair, laid out with the chunk's states. These cases put rows on both
strands of one position, more than 4 states at a position (the slot stride grows through the retry path) and a rows buffer that
has to grow, and compare the product with the oracle under the per-stage, MKP_FUSED=1 and MKP_TILE=1 kernels."""
import os

import pytest

from conftest import run_oracle, run_product, same_text
from test_gpu_parity import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[None, "MKP_FUSED", "MKP_TILE"], ids=["per_stage", "fused", "tile"])
def kernel_env(request):
    if request.param:
        os.environ[request.param] = "1"
    yield
    if request.param:
        os.environ.pop(request.param, None)


def both_strand_positions(bed_text):
    """positions (contig, start) with rows on both strands"""
    strands = {}
    for line in bed_text.splitlines():
        f = line.split("\t")
        strands.setdefault((f[0], f[1]), set()).add(f[5])
    return sum(1 for s in strands.values() if len(s) == 2)


def write_bed(path, contigs):
    # '.' intervals admit both strands at every position they hold
    with open(path, "w") as fh:
        for name, length in contigs:
            for k, s0 in enumerate(range(500, length - 1500, 3100)):
                fh.write("%s\t%d\t%d\tx\t0\t%s\n" % (name, s0, s0 + 900, ".+-"[k % 3]))


# (name, generator arguments, pileup flags, least number of positions with rows on both strands)
CASES = [
    # every position; duplex lists give 6 (base, code) states
    ("all_positions_duplex", ["--contig", "syn1:150000", "--coverage", 15, "--mods", "hma", "--duplex", "--seed", 71],
     ["--no-filtering"], 1000),
    # a motif whose reverse complement differs (CHH), a palindromic one with an offset, 6 states
    ("nonpalindromic_motifs", ["--contig", "syn1:150000", "--coverage", 15, "--mods", "hma", "--duplex", "--seed", 72],
     ["--motif", "CHH", "0", "--motif", "GATC", "1", "--motif", "A", "0", "--ref", "@FA", "-p", "0.2"], 0),
    # include-bed intervals on '+', '-' and both strands
    ("include_bed_both_strands", ["--contig", "c1:120000", "--contig", "c2:60000", "--coverage", 15, "--mods", "hma", "--duplex", "--seed", 73],
     ["--include-bed", "@BED", "--no-filtering"], 100),
    ("include_bed_cpg", ["--contig", "c1:120000", "--coverage", 15, "--mods", "hm", "--seed", 74],
     ["--include-bed", "@BED", "--cpg", "--ref", "@FA", "-p", "0.2"], 0),
]


@pytest.mark.parametrize("name,gen,flags,min_both", CASES, ids=[c[0] for c in CASES])
def test_strand_slots_match_oracle(name, gen, flags, min_both, native_lib, oracle_exe, synth_exe, tmp_path, kernel_env):
    prefix, info = synth(synth_exe, tmp_path, name, *gen)
    bed = str(tmp_path / "include.bed")
    write_bed(bed, [("c1", 120000), ("c2", 60000)])
    flags = [prefix + ".fa" if f == "@FA" else bed if f == "@BED" else f for f in flags]
    exp = run_oracle(oracle_exe, flags, prefix + ".bam", str(tmp_path / "o.bed"))
    rc, got = run_product(flags, prefix + ".bam", str(tmp_path / "g.bed"))
    assert rc == 0
    assert exp.count("\n") > 1000, "degenerate test input"
    assert both_strand_positions(exp) >= min_both
    assert same_text(got, exp)


def test_rows_buffer_grows(native_lib, oracle_exe, synth_exe, tmp_path, kernel_env):
    # the first chunks are tiny contigs (the rows buffer is sized from them), the later ones hold far more rows
    prefix, info = synth(synth_exe, tmp_path, "grow", "--contig", "t1:1500", "--contig", "t2:1500", "--contig", "big1:200000",
                         "--contig", "big2:150000", "--coverage", 20, "--mods", "hm", "--duplex", "--seed", 75)
    flags = ["--cpg", "--ref", prefix + ".fa"]
    exp = run_oracle(oracle_exe, flags, prefix + ".bam", str(tmp_path / "o.bed"))
    rc, got = run_product(flags, prefix + ".bam", str(tmp_path / "g.bed"))
    assert rc == 0
    small = sum(1 for line in exp.splitlines() if line.startswith("t"))
    assert 0 < small < 1024 and exp.count("\n") > 10 * 1024
    assert same_text(got, exp)
