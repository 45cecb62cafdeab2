"""`modkit sample-probs -o DIR --hist` of the product: thresholds.tsv and probabilities.tsv byte for byte against the CPU oracle
(its sample-probs report) and its restatement of the histogram table (tools/sample_hist_oracle.cpp) on the fixtures and a synthetic genome; the raw mkp_sample_mod_histogram counts against the wide arg-max histogram and, call
by call, against the independent model (callmodel.py); the two HTML pages against probabilities.tsv."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import FIX, GEN, ROOT
from test_call_table_cpu import CHEBI, build_table, model_run, write_table
from test_gpu_parity import synth
from test_sample_probs_hist_cpu import hist_oracle_exe, prob_to_qual  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

BAM = os.path.join(FIX, "bc_anchored_10_reads.sorted.bam")
MODKIT = os.path.join(ROOT, "modkit_b200", "_build", "modkit")
F32 = np.float32


def product_files(args, out):
    import modkit_b200
    rc = modkit_b200.sample_probs_main(["-o", str(out)] + [str(a) for a in args])
    assert rc == 0
    return {f: open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))}


def oracle_files(oracle_exe, hist_oracle_exe, args):
    """The two tables of the CPU restatements: the oracle's sample-probs report, and probabilities.tsv of the same sampled reads."""
    args = [str(a) for a in args]
    prefix = args[args.index("--prefix") + 1] + "_" if "--prefix" in args else ""
    run = lambda cmd: subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
    oracle_args = [a for i, a in enumerate(args) if a != "--hist" and a != "--prefix" and (i == 0 or args[i - 1] != "--prefix")]
    return {prefix + "probabilities.tsv": run([hist_oracle_exe] + args), prefix + "thresholds.tsv": run([oracle_exe, "sample-probs"] + oracle_args)}


def check_against_oracle(oracle_exe, hist_oracle_exe, args, tmp_path, tag):
    got = product_files(["--hist"] + args, tmp_path / ("p_" + tag))
    exp = oracle_files(oracle_exe, hist_oracle_exe, ["--hist"] + args)
    tables = {f: t for f, t in got.items() if f.endswith(".tsv")}
    assert tables == exp, args
    assert len(got) == 4 and sum(f.endswith(".html") for f in got) == 2
    assert exp[[f for f in exp if f.endswith("probabilities.tsv")][0]].count("\n") > 1
    return got


FIXTURE_CASES = {
    "default": [],
    "only_mapped": ["--only-mapped"],
    "edge_filter": ["--edge-filter", "50"],
    "ignore_h": ["--ignore", "h"],
    "region": ["--region", "oligo_1512_adapters:0-60"],
    "include_bed": ["--include-bed", os.path.join(FIX, "bc_anchored_10_reads_nofilt_cg_motif.bed")],
    "prefix": ["--prefix", "run1", "-p", "0.05,0.5"],
}


@pytest.mark.parametrize("case", sorted(FIXTURE_CASES))
def test_tables_match_oracle_on_fixture(case, native_lib, oracle_exe, hist_oracle_exe, tmp_path):
    got = check_against_oracle(oracle_exe, hist_oracle_exe, FIXTURE_CASES[case] + [BAM], tmp_path, case)
    if case == "prefix":
        assert sorted(got) == ["run1_counts.html", "run1_probabilities.tsv", "run1_proportion.html", "run1_thresholds.tsv"]


def test_tables_match_oracle_on_other_inputs(native_lib, oracle_exe, hist_oracle_exe, synth_exe, tmp_path):
    # all-context implicit fixture (inferred canonical entries), duplex fixture ('-' lists on C), a copy without index
    ecoli = os.path.join(GEN, "ecoli_reg.sorted.bam")
    got = check_against_oracle(oracle_exe, hist_oracle_exe, ["-n", "200", ecoli], tmp_path, "ecoli")
    probs = got["probabilities.tsv"].splitlines()
    assert any(ln.startswith("-\t") and ln.split("\t")[2] == "0.99609375" for ln in probs)     # bin 255: inferred entries at 1.0
    check_against_oracle(oracle_exe, hist_oracle_exe, ["--no-sampling", os.path.join(FIX, "duplex_modbam.sorted.bam")], tmp_path, "duplex")
    copy = str(tmp_path / "no_index.bam")
    shutil.copy(BAM, copy)
    a = check_against_oracle(oracle_exe, hist_oracle_exe, [copy], tmp_path, "noindex")
    b = product_files(["--hist", BAM], tmp_path / "with_index")
    assert a == b
    prefix, _ = synth(synth_exe, tmp_path, "s", "--contig", "c1:900000", "--contig", "c2:400000", "--coverage", 15, "--mods", "hma", "--odd-records", "--seed", 61)
    got = check_against_oracle(oracle_exe, hist_oracle_exe, ["-n", "400", prefix + ".bam"], tmp_path, "synth_n400")
    assert {ln.split("\t")[:2][0] for ln in got["probabilities.tsv"].splitlines()[1:]} >= {"-", "a", "h", "m"}
    check_against_oracle(oracle_exe, hist_oracle_exe, ["--no-sampling", prefix + ".bam"], tmp_path, "synth_all")


@pytest.fixture(scope="module")
def table_files(tmp_path_factory):
    table = build_table()
    bam, _ = write_table(table, tmp_path_factory.mktemp("histtable_gpu"))
    return table, bam


def state_code(key):
    key = int(key) & 0xffffffff
    return key & 0x7fffffff if key & 0x80000000 else chr(key)


@pytest.mark.parametrize("ignore", [None, "h", "m", CHEBI])
def test_raw_histogram_equals_model_call_by_call(ignore, table_files, native_lib):
    import modkit_b200
    table, bam = table_files
    calls, _, _ = model_run(table, ["--no-filtering"] + (["--ignore", ignore] if ignore else []))
    exp = {}
    n_off_grid = 0
    for _, _, (kind, code, v), _ in calls.values():
        k = (code if kind == "mod" else None, prob_to_qual(v))
        exp[k] = exp.get(k, 0) + 1
        n_off_grid += F32(v * F32(1024.0)) != np.rint(F32(v * F32(1024.0)))
    b = modkit_b200.Bam(bam, threads=4)
    ctx = modkit_b200.Context(0)
    code = 0 if ignore is None else ord(ignore) if not ignore.isdigit() else 0x80000000 | int(ignore)
    ctx.set_params(modkit_b200.make_params(numeric_mode=2 if ignore else 0, collapse_code=code))
    ctx.upload(b.pack(0, 0, b.refs[0][1]))
    hist, states = ctx.sample_mod_histogram()
    got = {}
    for s, q in zip(*np.nonzero(hist[1])):
        got[(None if s == 0 else state_code(states[s - 1]), int(q))] = int(hist[1, s, q])
    assert hist[0].sum() == hist[2].sum() == hist[3].sum() == 0
    assert all(int(states[s - 1]) >> 32 == 1 for s in range(1, 33) if hist[1, s].any())
    assert got == exp
    # every arg-max value off the 1/1024 grid (ReDistribute shares of 1/3) still lands in floor(v * 256)
    assert (ignore is None) == (n_off_grid == 0)
    wide, _, inexact = ctx.sample_histogram(wide=True)
    assert inexact == n_off_grid
    if inexact == 0:
        # on the grid, the arg-max histogram rebinned to prob_to_qual: bin k (k/1024) -> min(255, k >> 2)
        for base in range(4):
            rebinned = np.zeros(256, dtype=np.uint64)
            np.add.at(rebinned, np.minimum(255, np.arange(modkit_b200.HIST_BINS) >> 2), wide[base])
            assert (hist[base].sum(axis=0) == rebinned).all(), base
        assert hist[1, 0, 255] > 0 and wide[1, 1025:].sum() > 0


def test_off_grid_values_fail_and_write_nothing(table_files, native_lib, tmp_path):
    import modkit_b200
    _, bam = table_files
    out = tmp_path / "out"
    assert modkit_b200.sample_probs_main(["-o", str(out), "--hist", "--no-sampling", "--ignore", "h", bam]) == 1
    assert not out.exists()


def chart(html):
    line = [ln for ln in html.splitlines() if ln.strip().startswith("var option = ")][0]
    return json.loads(line.strip()[len("var option = "):-1])


def test_html_pages_match_probabilities(native_lib, tmp_path):
    import modkit_b200
    for colours, want in (([], {"C:-": "#0000FF", "C:h": "#FF00FF", "C:m": "#FF0000"}),
                          (["--dna-color", "C", "#123456", "--mod-color", "h", "#abcdef"], {"C:-": "#123456", "C:h": "#abcdef", "C:m": "#FF0000"})):
        out = tmp_path / ("c%d" % len(colours))
        got = product_files(["--hist", "--no-sampling"] + colours + [BAM], out)
        rows = [ln.split("\t") for ln in got["probabilities.tsv"].splitlines()[1:]]
        series = {}
        for code, base, start, _, n, _, _ in rows:
            series.setdefault(base + ":" + code, {})[int(F32(start) * F32(256.0))] = int(n)
        bins = sorted({q for s in series.values() for q in s})
        cats = ["[%s, %s)" % (modkit_b200.pct2(F32(q) / F32(256.0) * F32(100.0)), modkit_b200.pct2(F32(q + 1) / F32(256.0) * F32(100.0))) for q in bins]
        counts, props = chart(got["counts.html"]), chart(got["proportion.html"])
        assert counts["title"]["text"] == "Counts" and props["title"]["text"] == "Proportion"
        for c in (counts, props):
            assert c["xAxis"]["data"] == cats
            assert [s["name"] for s in c["series"]] == list(series)
            assert c["color"] == [want[name] for name in series]
        for s, p in zip(counts["series"], props["series"]):
            exp = [series[s["name"]].get(q, 0) for q in bins]
            assert s["data"] == exp
            tot = F32(sum(exp))
            assert [F32(x) for x in p["data"]] == [F32(F32(x) / tot) for x in exp]
        assert 'src="https://cdn.jsdelivr.net/npm/echarts' in got["counts.html"]


def test_force_overwrites_and_stdout_stays_empty(native_lib, oracle_exe, hist_oracle_exe, tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    for f in ("thresholds.tsv", "probabilities.tsv", "counts.html", "proportion.html"):
        (out / f).write_text("old\n")
    p = subprocess.run([MODKIT, "sample-probs", "-o", str(out), "--hist", "--force", BAM], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout == "", p.stderr
    exp = oracle_files(oracle_exe, hist_oracle_exe, ["--hist", BAM])
    for f, text in exp.items():
        assert (out / f).read_text() == text
    assert all((out / f).read_text() != "old\n" for f in os.listdir(out))
    # -o without --hist: only thresholds.tsv, the table that goes to stdout without -o
    only = tmp_path / "only"
    p = subprocess.run([MODKIT, "sample-probs", "-o", str(only), BAM], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout == ""
    assert os.listdir(only) == ["thresholds.tsv"]
    assert (only / "thresholds.tsv").read_text() == subprocess.run([MODKIT, "sample-probs", BAM], capture_output=True, text=True, check=True).stdout
