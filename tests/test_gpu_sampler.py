"""The threshold sampler reads its candidates from one of three sources: the index fetch (device ingest of an indexed BAM, sampler
beside the load), the records resident on the host (--host-ingest, the size fallback) and the records resident on the device
(a BAM without index). Every source must select the reads the oracle selects: same estimated thresholds, same bedMethyl, and
for `summary` the same call counts and `total_reads_used`."""
import shutil
import struct
import subprocess

import pytest

import bamio
from test_gpu_parity import synth
from test_gpu_summary import oracle as oracle_report, product as product_report
from test_hemi_cpu import hemi_oracle_exe  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

GENOME = ["--contig", "c1:200000", "--contig", "c2:90000", "--contig", "c3:40000", "--contig", "c4:150000", "--coverage", 10, "--mean-len", 4000,
          "--mods", "hm", "--odd-records", "--seed", 71]


def with_unplaced(prefix):
    """The genome's BAM plus unmapped reads without coordinates (copies of every 8th forward read, MM/ML kept), re-indexed."""
    b = bamio.Bam(prefix + ".bam")
    extra = []
    for i, r in enumerate(b.records):
        f = bamio.rec_fields(r)
        mm, ml = bamio.get_aux(r, b"MM"), bamio.get_aux(r, b"ML")
        if i % 8 or f["tid"] < 0 or f["flag"] & 0xf14 or mm is None or ml is None:
            continue
        seq = "".join(bamio.SEQ_NIB[(f["seq"][k >> 1] >> (0 if k & 1 else 4)) & 15] for k in range(f["l_seq"]))
        extra.append(bamio.make_record(-1, -1, 4, [], seq, mm=mm, ml=list(ml), name="u%d" % i))
    assert len(extra) > 20
    out = bamio.bam_of(b.refs, b.records + extra, b.header_text)
    out.write(prefix + ".bam", index=True)


@pytest.fixture(scope="module")
def genome(synth_exe, tmp_path_factory):
    d = tmp_path_factory.mktemp("sampler")
    prefix, _ = synth(synth_exe, d, "g", *GENOME)
    with_unplaced(prefix)
    noidx = str(d / "noidx.bam")
    shutil.copy(prefix + ".bam", noidx)
    with open(str(d / "inc.bed"), "w") as f:
        for name, a, b in (("c1", 10000, 60000), ("c1", 120000, 125000), ("c2", 0, 90000), ("c4", 70000, 140000)):
            f.write("%s\t%d\t%d\n" % (name, a, b))
    return prefix, noidx, str(d / "inc.bed")


def oracle_thresholds(stderr):
    return {ln.split()[-1].rstrip("."): ln.split()[4] for ln in stderr.splitlines() if ln.startswith("> Using filter threshold")}


def product_run(args, bam, out, hemi=False):
    """One in-process run; returns (text, {base: "%.9g" threshold}) from the run's stats."""
    import modkit_b200
    tail = ["--quiet", bam] + (["-o", out] if hemi else [out])
    rc, st = modkit_b200.pileup_main_sharded(list(args) + tail, 0, 1, None, hemi=hemi)
    assert rc == 0, args
    thr = {b: "%.9g" % st["threshold_" + b] for b in "ACGT" if st["threshold_" + b] >= 0}
    return open(out).read(), thr


def devices_run(args, bam, out, hemi=False):
    import modkit_b200
    rc = (modkit_b200.pileup_hemi_main if hemi else modkit_b200.pileup_main)(list(args) + ["--devices", "0,0", "--quiet", bam] + (["-o", out] if hemi else [out]))
    assert rc == 0, args
    return open(out).read()


CASES = [
    ("small_groups_merge", ["-n", "150", "--sampling-interval-size", "15000"]),
    ("quota_capped", ["-n", "100000"]),
    ("sample_all", ["-f", "1.0", "--sampling-interval-size", "50000"]),
    ("include_unmapped", ["--include-unmapped", "-n", "400"]),
    ("regions", ["--region", "c1:20000-180000", "--sample-region", "c4:10000-120000", "-n", "300"]),
    ("include_bed", ["--include-bed", "@BED", "-n", "500"]),
    ("edge_filter", ["--edge-filter", "20,30", "-n", "500"]),
]


@pytest.mark.parametrize("name,flags", CASES, ids=[c[0] for c in CASES])
def test_every_source_selects_the_oracle_reads(name, flags, genome, native_lib, oracle_exe, tmp_path):
    prefix, noidx, bed = genome
    flags = [bed if f == "@BED" else f for f in flags]
    p = subprocess.run([oracle_exe, "pileup", "-t", "4"] + flags + [prefix + ".bam", str(tmp_path / "o.bed")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    exp, exp_thr = open(str(tmp_path / "o.bed")).read(), oracle_thresholds(p.stderr)
    assert exp_thr and exp.count("\n") > 1000
    for src, extra, bam in (("index", [], prefix + ".bam"), ("host", ["--host-ingest"], prefix + ".bam"), ("device", [], noidx)):
        got, thr = product_run(flags + extra, bam, str(tmp_path / (src + ".bed")))
        assert thr == exp_thr, src
        assert got == exp, src
    assert devices_run(flags, prefix + ".bam", str(tmp_path / "d.bed")) == exp


def test_hemi_sources_select_the_oracle_reads(native_lib, hemi_oracle_exe, synth_exe, tmp_path):
    prefix, _ = synth(synth_exe, tmp_path, "d", "--contig", "d1:150000", "--contig", "d2:60000", "--coverage", 10, "--mean-len", 4000, "--mods", "hm",
                      "--duplex", "--seed", 73)
    noidx = str(tmp_path / "noidx.bam")
    shutil.copy(prefix + ".bam", noidx)
    flags = ["-r", prefix + ".fa", "--cpg", "-n", "200", "--sampling-interval-size", "20000"]
    p = subprocess.run([hemi_oracle_exe, "pileup-hemi", "-t", "4", prefix + ".bam"] + flags + ["-o", str(tmp_path / "o.bed")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    exp, exp_thr = open(str(tmp_path / "o.bed")).read(), oracle_thresholds(p.stderr)
    assert exp_thr and exp.count("\n") > 200
    for src, extra, bam in (("index", [], prefix + ".bam"), ("host", ["--host-ingest"], prefix + ".bam"), ("device", [], noidx)):
        got, thr = product_run(flags + extra, bam, str(tmp_path / (src + ".bed")), hemi=True)
        assert thr == exp_thr, src
        assert got == exp, src
    assert devices_run(flags, prefix + ".bam", str(tmp_path / "d.bed"), hemi=True) == exp


def test_summary_with_and_without_index(genome, native_lib, oracle_exe, tmp_path):
    prefix, noidx, _ = genome
    for args in (["--tsv", "-n", "300", "-i", "20000"], ["--tsv", "-n", "250", "--only-mapped"]):
        exp = oracle_report(oracle_exe, "summary", args + [prefix + ".bam"])
        assert "total_reads_used" in exp
        assert product_report("summary", args + [prefix + ".bam"], tmp_path) == exp
        assert product_report("summary", args + [noidx], tmp_path) == exp


def test_size_fallback_keeps_the_sampler_reader(genome, native_lib, oracle_exe, tmp_path, monkeypatch):
    """A BAM whose contigs are not stored in header order cannot be loaded range by range; with a tiny device budget the run
    reads it on the host while the sampler, already started, keeps fetching through the index."""
    import json
    prefix, _, _ = genome
    b = bamio.Bam(prefix + ".bam")
    tid = lambda r: struct.unpack_from("<i", r, 0)[0]
    order = {1: 0, 0: 1}                       # c2's records first, then c1, c3, c4 and the unplaced reads
    b.records = sorted(b.records, key=lambda r: order.get(tid(r), tid(r) % (1 << 31)))
    swapped = str(tmp_path / "swapped.bam")
    b.write(swapped, index=True)
    flags = ["-n", "400", "--include-unmapped"]
    p = subprocess.run([oracle_exe, "pileup", "-t", "4"] + flags + [swapped, str(tmp_path / "o.bed")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    exp, exp_thr = open(str(tmp_path / "o.bed")).read(), oracle_thresholds(p.stderr)
    host, host_thr = product_run(flags + ["--host-ingest"], swapped, str(tmp_path / "h.bed"))
    monkeypatch.setenv("MODKIT_B200_INGEST_BUDGET_MB", "1")
    sj = str(tmp_path / "s.json")
    got, thr = product_run(flags + ["--stats-json", sj], swapped, str(tmp_path / "f.bed"))
    assert json.load(open(sj))["ingest"] == "host"
    assert thr == host_thr == exp_thr
    assert got == host == exp


def test_summary_rejects_a_repeated_base_threshold(genome, native_lib, tmp_path, capfd):
    import modkit_b200
    prefix, _, _ = genome
    rc = modkit_b200.summary_main(["--filter-threshold", "C:0.5", "--filter-threshold", "C:0.6", prefix + ".bam", "--out", str(tmp_path / "r.txt")])
    assert rc == 1
    assert "repeated threshold for base C" in capfd.readouterr().err
