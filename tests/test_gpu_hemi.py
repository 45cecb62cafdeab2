"""`pileup-hemi` on the GPU (k_parse / k_resolve, k_hemi_count, k_hemi_rows through the in-process CLI): the reference's
goldens, the CPU oracle on seeded synthetic duplex genomes (forward and reverse reads, reads without usable tags), and
invariance of the output under the chunk size, the ingest path and the number of devices. Bit-exact text everywhere."""
import json
import os
import subprocess

import pytest

from conftest import GEN
from test_hemi_cpu import BAM, FA, GOLDENS, REGION, hemi_oracle_exe  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu


def run_hemi(args, out=None):
    """In-process `modkit pileup-hemi` on cuda:0; returns (exit code, text)."""
    import modkit_b200
    rc = modkit_b200.pileup_hemi_main(list(args) + ["--quiet"] + (["-o", out] if out else []))
    return rc, (open(out).read() if out and os.path.isfile(out) else "")


def run_oracle_hemi(exe, args, out):
    p = subprocess.run([exe, "pileup-hemi", "-t", "4"] + list(args) + ["-o", out], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    return open(out).read()


def synth(synth_exe, tmp_path, name, *args):
    prefix = str(tmp_path / name)
    out = subprocess.run([synth_exe, "--out", prefix, "--threads", "4"] + [str(a) for a in args], capture_output=True, text=True, check=True)
    return prefix, json.loads(out.stdout)


@pytest.mark.parametrize("golden,flags", GOLDENS, ids=[g[0] for g in GOLDENS])
def test_gpu_hemi_matches_reference_golden(golden, flags, native_lib, tmp_path):
    rc, got = run_hemi([BAM, "-r", FA, "--region", REGION] + flags, str(tmp_path / "g.bed"))
    assert rc == 0 and got == open(os.path.join(GEN, golden)).read()


DUPLEX = ["--contig", "c1:250000", "--contig", "c2:120000", "--coverage", 15, "--mods", "hma", "--duplex"]
HEMI_CASES = [
    ("default", DUPLEX + ["--seed", 51], ["--cpg"]),
    ("no_filtering", DUPLEX + ["--seed", 52], ["--cpg", "--no-filtering"]),
    ("thresholds", DUPLEX + ["--seed", 53], ["--cpg", "--filter-threshold", "C:0.7", "--filter-threshold", "A:0.6", "--mod-thresholds", "h:0.8"]),
    ("ignore_h", DUPLEX + ["--seed", 54], ["--cpg", "--ignore", "h"]),
    ("combine_mods", DUPLEX + ["--seed", 55], ["--cpg", "--combine-mods", "--mixed-delim"]),
    ("edge_filter", DUPLEX + ["--seed", 56], ["--cpg", "--edge-filter", "100,40", "-p", "0.2"]),
    ("edge_filter_inverted", DUPLEX + ["--seed", 57], ["--cpg", "--edge-filter", "500", "--invert-edge-filter", "--no-filtering"]),
    ("max_depth", ["--contig", "c1:150000", "--coverage", 30, "--mods", "hm", "--duplex", "--seed", 58, "--start-grid", 2500],
     ["--cpg", "--max-depth", "12", "--filter-threshold", "C:0.7", "-i", "30000"]),
    ("include_bed", DUPLEX + ["--seed", 59], ["--cpg", "--include-bed", "@BED", "-p", "0.2"]),
    ("region", DUPLEX + ["--seed", 60], ["--cpg", "--region", "c1:20000-190000", "-i", "30011"]),
    ("implicit_forced", ["--contig", "c1:200000", "--coverage", 15, "--mods", "hm", "--duplex", "--implicit", "--seed", 61],
     ["--cpg", "--force-allow-implicit", "--no-filtering"]),
    ("motif_gatc_1", DUPLEX + ["--seed", 62], ["--motif", "GATC", "1", "--no-filtering"]),
    ("motif_ta_1_negative_partner", DUPLEX + ["--seed", 63], ["--motif", "TA", "1", "--filter-threshold", "A:0.6", "--filter-threshold", "C:0.7"]),
    ("soft_masked_k", DUPLEX + ["--seed", 64], ["--cpg", "-k", "--no-filtering", "@MASK"]),
    ("interval_25", DUPLEX + ["--seed", 65], ["--cpg", "-i", "25", "--no-filtering"]),
    ("interval_88", DUPLEX + ["--seed", 66], ["--cpg", "-i", "88", "-p", "0.2"]),
    ("interval_10000", DUPLEX + ["--seed", 67], ["--motif", "TA", "1", "-i", "10000", "--no-filtering"]),
]


def write_include_bed(path):
    with open(path, "w") as fh:     # stranded, unstranded (BED3) and overlapping intervals
        for name, length in (("c1", 250000), ("c2", 120000)):
            for k, s0 in enumerate(range(1000, length - 2000, 4700)):
                strand = "+-."[k % 3]
                fh.write("%s\t%d\t%d\n" % (name, s0, s0 + 900) if k % 5 == 4 else "%s\t%d\t%d\tx\t0\t%s\n" % (name, s0, s0 + 700 + 300 * (k % 2), strand))
                if k % 7 == 0:
                    fh.write("%s\t%d\t%d\tx\t0\t+\n" % (name, s0 + 500, s0 + 1500))


def soft_mask(fa_in, fa_out):
    """Lower-case every other 2 kb block of the reference (line layout and .fai stay valid)."""
    pos = 0
    with open(fa_in) as src, open(fa_out, "w") as dst:
        for line in src:
            if line.startswith(">"):
                pos = 0
                dst.write(line)
                continue
            s = line.rstrip("\n")
            dst.write("".join(c.lower() if ((pos + i) // 2000) % 2 else c for i, c in enumerate(s)) + "\n")
            pos += len(s)
    with open(fa_in + ".fai") as src, open(fa_out + ".fai", "w") as dst:
        dst.write(src.read())


@pytest.mark.parametrize("name,gen,flags", HEMI_CASES, ids=[c[0] for c in HEMI_CASES])
def test_gpu_hemi_matches_oracle_on_synthetic(name, gen, flags, native_lib, hemi_oracle_exe, synth_exe, tmp_path):
    prefix, _ = synth(synth_exe, tmp_path, name, *gen)
    fa = prefix + ".fa"
    if "@MASK" in flags:
        fa = str(tmp_path / "masked.fa")
        soft_mask(prefix + ".fa", fa)
        flags = [f for f in flags if f != "@MASK"]
    bed = str(tmp_path / "include.bed")
    write_include_bed(bed)
    args = [prefix + ".bam", "-r", fa] + [bed if f == "@BED" else f for f in flags]
    exp = run_oracle_hemi(hemi_oracle_exe, args, str(tmp_path / "o.bed"))
    rc, got = run_hemi(args, str(tmp_path / "g.bed"))
    assert rc == 0
    assert exp.count("\n") > 200, "degenerate test input"
    assert got == exp


def test_gpu_hemi_soft_mask_changes_focus(native_lib, synth_exe, tmp_path):
    # -k keeps the reference's case: lower-case CpGs are not motif hits
    prefix, _ = synth(synth_exe, tmp_path, "mask", *(DUPLEX + ["--seed", 68]))
    fa = str(tmp_path / "masked.fa")
    soft_mask(prefix + ".fa", fa)
    rc, upper = run_hemi([prefix + ".bam", "-r", fa, "--cpg", "--no-filtering"], str(tmp_path / "u.bed"))
    rc2, kept = run_hemi([prefix + ".bam", "-r", fa, "--cpg", "--no-filtering", "-k"], str(tmp_path / "k.bed"))
    assert rc == rc2 == 0 and 0 < kept.count("\n") < upper.count("\n")


def test_gpu_hemi_invariance(native_lib, synth_exe, tmp_path):
    """Chunk size, host versus device ingest, three shards on one device, stdout: the same text."""
    prefix, _ = synth(synth_exe, tmp_path, "inv", "--contig", "c1:400000", "--contig", "c2:150000", "--coverage", 15, "--mods", "hm",
                      "--duplex", "--seed", 69)
    base = [prefix + ".bam", "-r", prefix + ".fa", "--cpg", "-i", "10000"]
    rc, ref = run_hemi(base, str(tmp_path / "ref.bed"))
    assert rc == 0 and ref.count("\n") > 5000
    variants = [["--gpu-chunk-bp", "50000"], ["--gpu-chunk-bp", "130001"], ["--host-ingest"], ["--devices", "0,0,0"]]
    for k, extra in enumerate(variants):
        rc, got = run_hemi(base + extra, str(tmp_path / ("v%d.bed" % k)))
        assert rc == 0 and got == ref, extra


def test_gpu_hemi_stdout(native_lib, tmp_path):
    """Without -o the rows go to stdout (a child process, so its stdout can be read)."""
    import sys
    from conftest import ROOT
    code = "import sys; sys.path.insert(0, %r); import modkit_b200; sys.exit(modkit_b200.pileup_hemi_main(sys.argv[1:]))" % ROOT
    p = subprocess.run([sys.executable, "-c", code, BAM, "-r", FA, "--region", REGION, "--cpg", "--mixed-delim", "--quiet"],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert p.stdout == open(os.path.join(GEN, "duplex_hemi.bed")).read()


def test_gpu_hemi_row_api(native_lib, hemi_oracle_exe, synth_exe, tmp_path):
    """The raw C-ABI pass: upload with the + strand CpG positions as focus_pos, mkp_hemi_resident, mkp_fetch_hemi_rows."""
    import numpy as np
    import modkit_b200
    prefix, _ = synth(synth_exe, tmp_path, "api", "--contig", "c1:100000", "--coverage", 15, "--mods", "hm", "--duplex", "--seed", 70)
    seq = "".join(ln.strip() for ln in open(prefix + ".fa") if not ln.startswith(">"))
    n_words = (100000 + 31) // 32
    fpos = np.zeros(n_words, dtype=np.uint32)
    for i in range(len(seq) - 1):
        if seq[i] == "C" and seq[i + 1] == "G":
            fpos[i >> 5] |= np.uint32(1 << (i & 31))
    bam = modkit_b200.Bam(prefix + ".bam", threads=4)
    pk = bam.pack(0, 0, 100000)
    fneg = np.zeros(n_words, dtype=np.uint32)
    ch = pk.chunk()
    ch.focus_pos = fpos.ctypes.data
    ch.focus_neg = fneg.ctypes.data
    ctx = modkit_b200.Context(0)
    ctx.set_params(modkit_b200.make_params(base_thresholds={"C": 0.7}))
    ctx._check(ctx._lib.mkp_upload_chunk(ctx._h, ch))
    st = ctx.hemi_resident([0], 1)
    rows = ctx.fetch_hemi_rows()
    assert st.n_rows == len(rows) > 1000 and (np.diff(rows["pos"].astype(np.int64)) >= 0).all()
    assert (rows["count"] > 0).all() and set(np.unique(rows["primary_base"])) <= {0, 1, 2, 3}
    exp = run_oracle_hemi(hemi_oracle_exe, [prefix + ".bam", "-r", prefix + ".fa", "--cpg", "--filter-threshold", "C:0.7", "-i", "100000"], str(tmp_path / "o.bed"))
    assert len(rows) == exp.count("\n")
