"""The call table (test_call_table_cpu.py) through the product: every called position's counts against the independent model
(callmodel.py) and the whole text against the oracle, for the default kernels and, with a motif so that their focus bitmaps
engage, the fused (MKP_FUSED=1) and tile (MKP_TILE=1) kernels; the raw arg-max histogram bin for bin; summary,
sample-probs, pileup-hemi on the duplex variant and a two-rank run of the estimated threshold. Arg-max values above 1.0
(ML sums up to 1.01, ReDistribute shares) are legal and must estimate a threshold; values off the 1/1024 grid fail loudly."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import callmodel as cm
from conftest import ROOT, run_oracle, run_product, same_text
from test_call_table_cpu import (CHEBI, Read, Table, build_table, check_rows_against_model, f32_text, flag_sets, model_run,
                                 write_table)
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

FOCUS = ["no_filtering", "C_384_512_above", "mod_anymod_C", "ignore_m", "ignore_chebi", "combine_mods", "estimated_p01", "traditional"]


@pytest.fixture(scope="module")
def table_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("calltable")
    table = build_table()
    bam, fa = write_table(table, d)
    return table, bam, fa


@pytest.fixture(scope="module")
def two_code_files(tmp_path_factory):
    """The table without its three- and four-code reads: every arg-max value on the 1/1024 grid under --ignore h, so that
    --preset traditional estimates its threshold (values above 1.0 included)."""
    d = tmp_path_factory.mktemp("twocode")
    table = build_table(multi=False)
    bam, fa = write_table(table, d)
    return table, bam, fa


@functools.lru_cache(maxsize=None)
def oracle_text(oracle_exe, flags, bam, out):
    return run_oracle(oracle_exe, list(flags), bam, out)


def with_env(kernel, fn):
    if kernel:
        os.environ[kernel] = "1"
    try:
        return fn()
    finally:
        os.environ.pop(kernel or "", None)


@pytest.mark.parametrize("name", [n for n, _ in flag_sets(build_table(), "FA")])
def test_pileup_matches_model_and_oracle(name, table_files, two_code_files, native_lib, oracle_exe, tmp_path_factory):
    flags = dict(flag_sets(table_files[0], table_files[2]))[name]
    table, bam, fa = two_code_files if name == "traditional" else table_files
    flags = [fa if f == table_files[2] else f for f in flags]
    d = tmp_path_factory.mktemp(name)
    runs = [(None, flags)]
    if name in FOCUS:
        focus = flags if name == "traditional" else flags + ["--motif", "C", "0", "--ref", fa]
        runs += [(k, focus) for k in ("MKP_FUSED", "MKP_TILE")]
    for kernel, fl in runs:
        exp = oracle_text(oracle_exe, tuple(fl), bam, str(d / ("o%d.bed" % len(fl))))
        rc, got = with_env(kernel, lambda: run_product(fl, bam, str(d / "g.bed")))
        assert rc == 0, (kernel, fl)
        check_rows_against_model(got, table, fl)
        assert same_text(got, exp), (kernel, fl)


@pytest.mark.parametrize("ignore", [None, "h", "m", CHEBI])
def test_sample_histogram_bins_equal_model(ignore, table_files, native_lib):
    """The raw arg-max histogram of every read: bin round(v * 1024) of each model value, values above 1.0 in their own bins of
    the wide histogram; off-grid values (ReDistribute dividing by 3) counted as inexact."""
    import modkit_b200
    table, bam, _ = table_files
    calls, failed, _ = model_run(table, ["--no-filtering"] + (["--ignore", ignore] if ignore else []))
    vals = np.array([a[2] for _, _, a, _ in calls.values()], dtype=np.float32)
    scaled = vals * np.float32(1024.0)
    bins = np.rint(scaled).astype(np.int64)
    off = int((bins.astype(np.float32) != scaled).sum())
    exp = np.bincount(bins, minlength=modkit_b200.HIST_BINS)
    b = modkit_b200.Bam(bam, threads=4)
    ctx = modkit_b200.Context(0)
    code = 0 if ignore is None else ord(ignore) if not ignore.isdigit() else 0x80000000 | int(ignore)     # ModCodeRepr as u32
    ctx.set_params(modkit_b200.make_params(numeric_mode=2 if ignore else 0, collapse_code=code))
    ctx.upload(b.pack(0, 0, b.refs[0][1]))
    wide, _, inexact = ctx.sample_histogram(wide=True)
    assert wide[0].sum() == wide[2].sum() == wide[3].sum() == 0
    assert (wide[1] == exp).all() and inexact == off
    assert (ignore is None) == (off == 0) and exp[1025:].sum() > 0
    narrow, _, inexact = ctx.sample_histogram()
    assert (narrow[1][:1024] == exp[:1024]).all() and narrow[1][1024] == exp[1024:].sum()
    assert inexact == off + exp[1025:].sum()


def test_reports_match_model_and_oracle(table_files, two_code_files, native_lib, oracle_exe, tmp_path):
    """summary and sample-probs; the estimated threshold under --ignore h on the two-code table (arg-max values above 1.0)."""
    from test_gpu_summary import oracle, product
    table, bam, _ = table_files
    two = two_code_files[1]
    for cmd, args in (("summary", ["--tsv", "--no-sampling", bam]), ("summary", ["--tsv", "--no-sampling", "--no-filtering", bam]),
                      ("summary", ["--tsv", "--no-sampling", "--ignore", "h", two]),
                      ("summary", ["--tsv", "--no-sampling", "--ignore", "m", "--filter-threshold", "C:" + f32_text(table.thresholds["m"]), bam]),
                      ("sample-probs", ["--no-sampling", "--ignore", "h", "-p", "0.5,0.999", two]),
                      ("sample-probs", ["--no-sampling", "-p", "0.1,0.5,0.9,0.999", bam])):
        exp = oracle(oracle_exe, cmd, args)
        assert product(cmd, args, tmp_path) == exp, (cmd, args)
    calls, _, _ = model_run(table, ["--no-filtering"])
    vals = [a[2] for _, _, a, _ in calls.values()]
    rows = [ln.split() for ln in exp.splitlines()[1:]]
    assert [np.float32(r[2]) for r in rows] == [cm.percentile(vals, q) for q in (0.1, 0.5, 0.9, 0.999)]


def test_hemi_duplex_table_matches_oracle(native_lib, hemi_oracle_exe, tmp_path):
    from test_gpu_hemi import run_hemi, run_oracle_hemi
    table = build_table(duplex=True)
    bam, fa = write_table(table, tmp_path, "duplex")
    for flags in (["--no-filtering"], ["--filter-threshold", "C:0.75"], ["--ignore", "h", "--filter-threshold", "C:" + f32_text(513 / 1024)], []):
        args = [bam, "-r", fa, "--cpg"] + flags
        exp = run_oracle_hemi(hemi_oracle_exe, args, str(tmp_path / "oh.bed"))
        assert exp.count("\n") > 3000
        rc, got = run_hemi(args, str(tmp_path / "gh.bed"))
        assert rc == 0 and same_text(got, exp), flags


def test_two_ranks_estimate_the_same_threshold(two_code_files, native_lib, oracle_exe, tmp_path):
    """The estimated-threshold case on --devices 0,0: the ranks exchange the wide histograms and agree with one device."""
    table, bam, fa = two_code_files
    flags = ["--preset", "traditional", "--ref", fa]
    exp = oracle_text(oracle_exe, tuple(flags), bam, str(tmp_path / "o.bed"))
    rc, got = run_product(flags + ["--devices", "0,0"], bam, str(tmp_path / "g.bed"))
    assert rc == 0 and same_text(got, exp)
    check_rows_against_model(got, table, flags)


def test_off_grid_values_fail_loudly_without_output(native_lib, tmp_path):
    """Arg-max values off the 1/1024 grid (three codes, --ignore of one: a share of 1/3) have no exact histogram quantile:
    the estimated-threshold run stops with its message and writes no bedMethyl; an explicit threshold runs."""
    reads = [Read("multi_hmf", [("C+hmf?", {i: (20 + i, 41, 60) for i in range(30)})], 30, rev=False)]
    bam, _ = write_table(Table(reads, {}), tmp_path, "offgrid")
    vals = [a[2] for _, _, a, _ in model_run(Table(reads, {}), ["--no-filtering", "--ignore", "m"])[0].values()]
    assert any(np.rint(v * 1024) != v * np.float32(1024) for v in vals)
    out = tmp_path / "x.bed"
    code = "import sys; sys.path.insert(0, %r); import modkit_b200; sys.exit(modkit_b200.pileup_main(sys.argv[1:]))" % ROOT
    p = subprocess.run([sys.executable, "-c", code, "--ignore", "m", "--quiet", bam, str(out)], capture_output=True, text=True)
    assert p.returncode == 1 and "not multiples of 1/1024" in p.stderr, p.stderr[-400:]
    assert not out.exists() or out.stat().st_size == 0
    rc, text = run_product(["--ignore", "m", "--filter-threshold", "C:0.5"], bam, str(out))
    assert rc == 0 and text.count("\n") > 10
