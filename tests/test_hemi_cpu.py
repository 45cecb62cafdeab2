"""`pileup-hemi` on the CPU: the oracle (oracle/hemi.hpp, binary oracle/_build/modkit_oracle_hemi) against the reference's two
goldens (tests/test_pileup_hemi.rs, moved onto the shifted chr20 window of tests/golden/make_duplex_fixtures.py), and the
argument errors of the oracle and of the product CLI, which reports them before it opens a device."""
import os
import subprocess
import sys

import pytest

from conftest import GEN, ROOT

BAM = os.path.join(GEN, "duplex_window.bam")
FA = os.path.join(GEN, "duplex_window.fa")
REGION = "chr20:63,835-90,468"       # chr20:22,613,835-22,640,468 of the reference's tests, shifted by 22,550,000

GOLDENS = [
    ("duplex_hemi_nofilt.bed", ["--motif", "CG", "0", "--no-filtering", "--mixed-delim"]),   # test_pileup_hemi_hm
    ("duplex_hemi.bed", ["--cpg", "--mixed-delim"]),                                        # test_pileup_hemi_preset
]


@pytest.fixture(scope="session")
def hemi_oracle_exe():
    """The `pileup-hemi` oracle (oracle/hemi_main.cpp), built when missing or older than its sources."""
    d = os.path.join(ROOT, "oracle")
    exe = os.path.join(d, "_build", "modkit_oracle_hemi")
    srcs = [os.path.join(d, f) for f in os.listdir(d) if f.endswith((".cpp", ".hpp"))]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-pthread", os.path.join(d, "hemi_main.cpp"), "-o", exe, "-lz"])
    return exe


def run_oracle_hemi(exe, args):
    return subprocess.run([exe, "pileup-hemi", "-t", "4"] + list(args), capture_output=True, text=True)


@pytest.mark.parametrize("golden,flags", GOLDENS, ids=[g[0] for g in GOLDENS])
def test_oracle_hemi_matches_reference_golden(golden, flags, hemi_oracle_exe, tmp_path):
    out = str(tmp_path / "o.bed")
    p = run_oracle_hemi(hemi_oracle_exe, [BAM, "-o", out, "-r", FA, "--region", REGION] + flags)
    assert p.returncode == 0, p.stderr
    exp = open(os.path.join(GEN, golden)).read()
    assert open(out).read() == exp and exp.count("\n") > 250


def test_oracle_hemi_stdout(hemi_oracle_exe):
    p = run_oracle_hemi(hemi_oracle_exe, [BAM, "-r", FA, "--region", REGION, "--cpg", "--mixed-delim"])
    assert p.returncode == 0 and p.stdout == open(os.path.join(GEN, "duplex_hemi.bed")).read()


REJECTED = [["--preset", "traditional"], ["--combine-strands"], ["--bedgraph"], ["--with-header"], ["--header"],
            ["--prefix", "x"], ["--partition-tag", "HP"]]
MOTIF_ERRORS = [
    ([], "either --cpg or a --motif must be provided for pileup-hemi"),
    (["--motif", "CGA", "0"], "motif must be palindromic for pileup-hemi"),
    (["--motif", "CH", "0"], "motif must be palindromic for pileup-hemi"),
]


@pytest.mark.parametrize("flag", REJECTED, ids=[r[0] for r in REJECTED])
def test_oracle_hemi_rejects_pileup_only_flags(flag, hemi_oracle_exe):
    p = run_oracle_hemi(hemi_oracle_exe, [BAM, "-r", FA, "--cpg"] + flag)
    assert p.returncode != 0 and "unexpected argument '%s'" % flag[0] in p.stderr


@pytest.mark.parametrize("flags,msg", MOTIF_ERRORS, ids=["no_motif", "CGA", "CH"])
def test_oracle_hemi_motif_errors(flags, msg, hemi_oracle_exe):
    p = run_oracle_hemi(hemi_oracle_exe, [BAM, "-r", FA] + flags)
    assert p.returncode != 0 and msg in p.stderr


def product_cli(args):
    """The product's in-process `modkit pileup-hemi`, in a child process (its messages go to the child's stderr)."""
    code = "import sys; sys.path.insert(0, %r); import modkit_b200; sys.exit(modkit_b200.pileup_hemi_main(sys.argv[1:]))" % ROOT
    return subprocess.run([sys.executable, "-c", code] + list(args), capture_output=True, text=True)


@pytest.mark.parametrize("flag", REJECTED, ids=[r[0] for r in REJECTED])
def test_product_hemi_rejects_pileup_only_flags(flag, native_lib):
    p = product_cli([BAM, "-r", FA, "--cpg"] + flag)
    assert p.returncode == 2 and "unexpected argument '%s'" % flag[0] in p.stderr


@pytest.mark.parametrize("flags,msg", MOTIF_ERRORS, ids=["no_motif", "CGA", "CH"])
def test_product_hemi_motif_errors(flags, msg, native_lib):
    p = product_cli([BAM, "-r", FA] + flags)
    assert p.returncode == 1 and msg in p.stderr and "CUDA" not in p.stderr


def test_product_hemi_needs_reference_and_one_bam(native_lib):
    p = product_cli([BAM, "--cpg"])
    assert p.returncode == 1 and "--ref" in p.stderr
    p = product_cli([BAM, BAM, "-r", FA, "--cpg"])
    assert p.returncode == 2 and "unexpected argument" in p.stderr


def test_modkit_cli_has_pileup_hemi(native_lib):
    exe = os.path.join(ROOT, "modkit_b200", "_build", "modkit")
    p = subprocess.run([exe, "pileup-hemi", BAM, "-r", FA, "--motif", "CGA", "0"], capture_output=True, text=True)
    assert p.returncode == 1 and "motif must be palindromic for pileup-hemi" in p.stderr
