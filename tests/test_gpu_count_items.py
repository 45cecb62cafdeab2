"""The work items of k_count_bases: the part [r_lo, r_hi) of a read that one warp counts. The table built at upload is checked item
for item against a Python model of the packed chunk, for several window sizes and chunk origins. Then the rows under forced tiny
windows (MKP_COUNT_ITEM_BP = 32, 64, 96: nearly every seam lands inside a CIGAR op, a deletion, a reference skip or beside an
insertion) are checked against the oracle and the column model: on a synthetic genome of 100-200 kb reads on both strands, with
explicit and implicit MM lists, chunked at an origin off the 32-position word grid; on the pileup-columns corpus through the raw
C ABI; and on the read-shapes CIGAR cases."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, run_oracle, run_product, same_text
from test_gpu_parity import synth

pytestmark = pytest.mark.gpu

REF_OPS, QUERY_OPS = (0, 2, 3, 7, 8), (0, 1, 4, 7, 8)


def model_items(hdrs, heap, cs, ce, S):
    """{read, r_lo, op, q, r} of every item: the read's span clipped to [cs, ce) is one item when at most S long, else it is cut at
    cs + (a & ~31) + j * S (a: the clipped start relative to cs); op is the first op whose reference end is past r_lo."""
    out = []
    for ri, h in enumerate(hdrs):
        cig = np.frombuffer(heap[int(h["off"]):int(h["off"]) + 4 * int(h["n_cigar"])].tobytes(), dtype="<u4").astype(np.int64)
        op, ln = cig & 15, cig >> 4
        rl, ql = np.where(np.isin(op, REF_OPS), ln, 0), np.where(np.isin(op, QUERY_OPS), ln, 0)
        r0 = int(h["ref_start"]) + np.cumsum(rl) - rl
        q0 = np.cumsum(ql) - ql
        lo, hi = max(int(h["ref_start"]), cs), min(int(h["ref_start"]) + int(rl.sum()), ce)
        if lo >= hi:
            continue
        a, b = lo - cs, hi - cs
        n = 1 if b - a <= S else (b - 1 - (a & ~31)) // S + 1
        for s in [lo] + [cs + (a & ~31) + j * S for j in range(1, n)]:
            k = int(np.nonzero((rl > 0) & (r0 <= s) & (s < r0 + rl))[0][0])
            out.append((ri, s, k, int(q0[k]), int(r0[k])))
    return np.array(out, dtype=np.uint32).reshape(-1, 5)


@pytest.fixture(scope="module")
def long_reads(synth_exe, tmp_path_factory):
    return synth(synth_exe, tmp_path_factory.mktemp("long"), "long", "--contig", "syn1:900000", "--coverage", 8, "--mean-len", 100000,
                 "--mods", "hm", "--seed", 91)[0]


@pytest.mark.parametrize("bp", [32, 96, 8192, None], ids=["32", "96", "8192", "default"])
@pytest.mark.parametrize("cs,ce", [(0, 900000), (12345, 250001), (100007, 165543)])
def test_item_table_matches_model(bp, cs, ce, long_reads, native_lib, monkeypatch):
    import modkit_b200
    if bp:
        monkeypatch.setenv("MKP_COUNT_ITEM_BP", str(bp))
    ctx = modkit_b200.Context(0)
    bam = modkit_b200.Bam(long_reads + ".bam", ctx=ctx)
    try:
        assert bam.device_chunk(0, cs, ce) > 0
        got = ctx.fetch_count_items()
        hdrs, heap = ctx.fetch_chunk()
    finally:
        bam.close()
        ctx.close()
    S = bp or 32768
    exp = model_items(hdrs, heap, cs, ce, S)
    assert len(exp) > len(hdrs) // 2
    assert got.shape == exp.shape and (got == exp).all()
    # items of one read tile its clipped span; seams lie on the chunk's word grid
    seam = (exp[1:, 0] == exp[:-1, 0])
    assert ((exp[1:, 1][seam] - cs) % 32 == 0).all()
    assert (exp[1:, 1][seam] - exp[:-1, 1][seam] <= S).all()


def test_bad_window_is_an_error(long_reads, native_lib, monkeypatch):
    import modkit_b200
    monkeypatch.setenv("MKP_COUNT_ITEM_BP", "100")
    ctx = modkit_b200.Context(0)
    bam = modkit_b200.Bam(long_reads + ".bam", ctx=ctx)
    try:
        with pytest.raises(modkit_b200.MkpError):
            bam.device_chunk(0, 0, 900000)
    finally:
        bam.close()
        ctx.close()


LONG_CASES = [
    ("explicit_all_positions", ["--mods", "hm", "--seed", 92], ["--no-filtering"]),
    ("explicit_cpg_combine", ["--mods", "hm", "--seed", 93], ["--cpg", "--combine-strands", "--ref", "@FA", "-p", "0.2"]),
    ("implicit_all_positions", ["--mods", "m", "--implicit", "--seed", 94], ["--no-filtering"]),
    ("implicit_edge_filter", ["--mods", "hm", "--implicit", "--seed", 95], ["--edge-filter", "500,300", "-p", "0.2"]),
]


@pytest.mark.parametrize("name,gen,flags", LONG_CASES, ids=[c[0] for c in LONG_CASES])
def test_long_reads_under_tiny_windows_match_oracle(name, gen, flags, native_lib, oracle_exe, synth_exe, tmp_path, monkeypatch):
    prefix, _ = synth(synth_exe, tmp_path, name, "--contig", "syn1:700000", "--coverage", 10, "--mean-len", 150000, *gen)
    flags = [prefix + ".fa" if f == "@FA" else f for f in flags]
    exp = run_oracle(oracle_exe, flags, prefix + ".bam", str(tmp_path / "o.bed"))
    assert exp.count("\n") > 10000, "degenerate test input"
    rc, got = run_product(flags, prefix + ".bam", str(tmp_path / "g.bed"))
    assert rc == 0 and same_text(got, exp)
    for bp in ("32", "96"):
        monkeypatch.setenv("MKP_COUNT_ITEM_BP", bp)
        rc, got = run_product(flags + ["--gpu-chunk-bp", "230017"], prefix + ".bam", str(tmp_path / ("g%s.bed" % bp)))
        assert rc == 0 and same_text(got, exp), bp


@pytest.mark.parametrize("bp", ["32", "64", "96"])
def test_corpora_under_tiny_windows(bp):
    """The raw C ABI cases of the pileup-columns corpus and the CIGAR cases of the read-shapes reads (every op, long CIGARs in
    CG:B,I), rerun with every read cut into windows of `bp` reference bases."""
    tests = [os.path.join(ROOT, "tests", f) for f in ("test_gpu_pileup_columns.py", "test_gpu_read_shapes.py")]
    env = dict(os.environ, MKP_COUNT_ITEM_BP=bp, PYTHONNOUSERSITE="1")
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-m", "gpu",
                        "-k", "raw_abi or cigar"] + tests, cwd=ROOT, env=env, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
