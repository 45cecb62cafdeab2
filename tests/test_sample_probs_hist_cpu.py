"""`sample-probs -o DIR --hist` without a GPU: the CPU restatement's probabilities.tsv (tools/sample_hist_oracle.cpp, on the
oracle's sampler and decode) on the call table against the independent model (callmodel.py), the host's probabilities.tsv
formatter against a float32 model of the reference's fold, and the argument and overwrite checks, which run before any device
work."""
import os
import subprocess

import numpy as np
import pytest

import callmodel as cm
from conftest import FIX, ROOT
from test_call_table_cpu import CHEBI, build_table, f32_text, write_table

F32 = np.float32
BAM = os.path.join(FIX, "bc_anchored_10_reads.sorted.bam")
MODKIT = os.path.join(ROOT, "modkit_b200", "_build", "modkit")


def prob_to_qual(v):
    """mod_bam.rs:798-806: exactly 1.0 -> 255, else floor(v * 256) in f32 with a saturating `as u8`."""
    v = F32(v)
    if v == F32(1.0):
        return 255
    s = np.floor(F32(v * F32(256.0)))
    return 0 if not s > 0 else 255 if s >= 255 else int(s)


def state_sort_key(code):
    """BaseState's derived Ord: Canonical, then Modified(Code(char)) by char, then Modified(ChEbi(u32)) by number."""
    return (0, 0) if code is None else (1, ord(code)) if isinstance(code, str) else (2, code)


def model_tsv(counts):
    """probabilities.tsv from {(base, code or None): {qual: n}} (ProbHistogram::get_artifacts, src/writers.rs:837-945)."""
    out = ["code\tprimary_base\trange_start\trange_end\tcount\tfrac\tpercentile_rank"]
    for (base, code) in sorted(counts, key=lambda k: ("ACGT".index(k[0]), state_sort_key(k[1]))):
        bins = counts[(base, code)]
        total = F32(sum(bins.values()))
        cum = F32(0.0)
        for q in sorted(bins):
            n = F32(bins[q])
            cum = F32(cum + n)
            rank = F32(F32(F32(cum - F32(F32(0.5) * n)) / total) * F32(100.0))
            out.append("\t".join(["-" if code is None else str(code), base, f32_text(F32(q) / F32(256.0)), f32_text(F32(q + 1) / F32(256.0)),
                                  str(bins[q]), f32_text(F32(n / total)), f32_text(rank)]))
    return "\n".join(out) + "\n"


@pytest.fixture(scope="session")
def hist_oracle_exe():
    """The probabilities.tsv restatement (tools/sample_hist_oracle.cpp), built when missing or older than its sources."""
    src = os.path.join(ROOT, "tools", "sample_hist_oracle.cpp")
    exe = os.path.join(ROOT, "tools", "_build", "sample_hist_oracle")
    d = os.path.join(ROOT, "oracle")
    srcs = [src] + [os.path.join(d, f) for f in os.listdir(d) if f.endswith(".hpp")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        os.makedirs(os.path.dirname(exe), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-pthread", src, "-o", exe, "-lz"])
    return exe


@pytest.fixture(scope="module")
def table_bam(tmp_path_factory):
    table = build_table()
    bam, _ = write_table(table, tmp_path_factory.mktemp("histtable"))
    return table, bam


@pytest.mark.parametrize("ignore", [None, "h", "m", CHEBI])
def test_oracle_probabilities_match_model(ignore, table_bam, hist_oracle_exe):
    table, bam = table_bam
    counts = {}
    above_one = 0
    for r in table.reads:
        res = cm.read_calls(r.model_lists(), cm.Caller(), ignore)
        for _, (kind, code, v), _ in (res or {}).values():
            q = prob_to_qual(v)
            above_one += v > 1.0
            counts.setdefault(("C", code if kind == "mod" else None), {})
            counts[("C", code if kind == "mod" else None)][q] = counts[("C", code if kind == "mod" else None)].get(q, 0) + 1
    flags = ["--no-sampling"] + (["--ignore", ignore] if ignore else [])
    got = subprocess.run([hist_oracle_exe] + flags + [bam], capture_output=True, text=True, check=True).stdout
    assert got == model_tsv(counts)
    assert above_one > 0 and 255 in counts[("C", None if ignore == "m" else "m")]
    if ignore != CHEBI:
        assert ("C", int(CHEBI)) in counts and got.rstrip().splitlines()[-1].startswith(CHEBI + "\t")


def test_formatter_matches_f32_fold_with_large_counts(native_lib):
    import modkit_b200
    rng = np.random.default_rng(5)
    hist = np.zeros((4, 33, 256), dtype=np.uint64)
    states = np.full(32, 0xffffffffffffffff, dtype=np.uint64)
    # state ids in registry order, not in row order: ChEBI before h before m
    states[0] = (1 << 32) | 0x80000000 | 76792
    states[1] = (1 << 32) | ord("h")
    states[2] = (1 << 32) | ord("m")
    states[3] = (0 << 32) | ord("a")
    big = [(1 << 24) - 1, 1 << 24, (1 << 24) + 1, (1 << 24) + 3, 3 << 24, (1 << 31) + 7, (1 << 40) + 1]
    for b, s in ((1, 0), (1, 1), (1, 2), (1, 3), (0, 0), (0, 4), (3, 0)):
        qs = rng.choice(256, size=40, replace=False)
        hist[b, s, qs] = rng.choice(big + [1, 2, 3, 1000], size=40)
    hist[2, 0, 255] = 1
    counts = {}
    for b in range(4):
        for s in range(33):
            nz = np.nonzero(hist[b, s])[0]
            if len(nz):
                code = None if s == 0 else int(states[s - 1] & 0x7fffffff) if states[s - 1] & 0x80000000 else chr(int(states[s - 1] & 0xffffffff))
                counts[("ACGT"[b], code)] = {int(q): int(hist[b, s, q]) for q in nz}
    got = modkit_b200.probabilities_tsv(hist, states)
    assert got == model_tsv(counts)
    lines = got.splitlines()
    assert [ln.split("\t")[:2] for ln in lines[1:]][0] == ["-", "A"]
    c_codes = [ln.split("\t")[0] for ln in lines[1:] if ln.split("\t")[1] == "C"]
    assert c_codes == sorted(c_codes, key=lambda c: state_sort_key(None if c == "-" else int(c) if c.isdigit() else c))
    assert modkit_b200.probabilities_tsv(np.zeros((4, 33, 256), dtype=np.uint64), states) == "code\tprimary_base\trange_start\trange_end\tcount\tfrac\tpercentile_rank\n"


def modkit(*args):
    return subprocess.run([MODKIT, "sample-probs"] + [str(a) for a in args], capture_output=True, text=True)


USAGE_ERRORS = {
    "prefix_without_out_dir": (["--prefix", "p", BAM], "--prefix"),
    "force_without_out_dir": (["--force", BAM], "--force"),
    "hist_without_out_dir": (["--hist", BAM], "--hist"),
    "dna_color_without_hist": (["-o", "@OUT", "--dna-color", "C", "#000000", BAM], "--hist"),
    "mod_color_without_hist": (["-o", "@OUT", "--mod-color", "m", "#000000", BAM], "--hist"),
    "odd_colour_values": ([BAM, "-o", "@OUT", "--hist", "--dna-color", "C"], "invalid number of arguments"),
    "out_file_with_out_dir": (["-o", "@OUT", "--out", "@FILE", BAM], "cannot be used with"),
}


@pytest.mark.parametrize("case", sorted(USAGE_ERRORS))
def test_usage_errors(case, native_lib, tmp_path):
    args, message = USAGE_ERRORS[case]
    out, f = tmp_path / "out", tmp_path / "report.txt"
    args = [str(out) if a == "@OUT" else str(f) if a == "@FILE" else a for a in args]
    # clap's `requires` rules and conflicts are usage errors (exit 2), raised before anything is opened or created
    p = modkit(*args)
    assert p.returncode == 2 and message in p.stderr, p.stderr
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("flag,value,message", [("--dna-color", "CG", "DNA base should be a char"), ("--dna-color", "N", "invalid DNA base"),
                                                ("--dna-color", "c", "invalid DNA base"), ("--mod-color", "m1", "failed to parse mod code")])
def test_bad_colour_keys(flag, value, message, native_lib, tmp_path):
    # checked at run time, as the reference does, but before any device work
    out = tmp_path / "out"
    p = modkit("-o", out, "--hist", flag, value, "#123456", BAM)
    assert p.returncode == 1 and "> Error! " + message in p.stderr, p.stderr
    assert not out.exists()


@pytest.mark.parametrize("name", ["thresholds.tsv", "probabilities.tsv", "counts.html", "proportion.html"])
@pytest.mark.parametrize("prefix", [None, "run1"])
def test_refuses_to_overwrite(name, prefix, native_lib, tmp_path):
    out = tmp_path / "out"
    out.mkdir()
    fn = (prefix + "_" + name) if prefix else name
    (out / fn).write_text("keep me\n")
    p = modkit("-o", out, "--hist", *(["--prefix", prefix] if prefix else []), BAM)
    assert p.returncode == 1 and "refusing to overwrite" in p.stderr and fn in p.stderr, p.stderr
    assert os.listdir(out) == [fn] and (out / fn).read_text() == "keep me\n"
    if name == "thresholds.tsv":
        # without --hist only thresholds.tsv is checked
        p = modkit("-o", out, *(["--prefix", prefix] if prefix else []), BAM)
        assert p.returncode == 1 and "refusing to overwrite" in p.stderr
    else:
        # the histogram files are only checked with --hist, and a file of the other prefix does not count
        other = ["--prefix", "other"] if not prefix else []
        p = modkit("-o", out, "--hist", *other, "--region", "no_such_contig", BAM)
        assert "refusing to overwrite" not in p.stderr
    assert os.listdir(out) == [fn] and (out / fn).read_text() == "keep me\n"
