"""--partition-tag in interval-sharded runs: the ranks write the one-device directory (same file names, byte-identical files), as
threads of one process (`--devices`, works with one GPU) and as processes under torchrun over NCCL; partition tag values of any
length read on the GPU (mkp_bam_tag_values) against the host aux reader."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, read_dir, run_product
from test_gpu_parity import synth

pytestmark = pytest.mark.gpu

GENOME = ["--contig", "c1:400000", "--contig", "c2:160000", "--contig", "c3:90000", "--contig", "c4:250000", "--coverage", 15, "--mods", "hm",
          "--seed", 52, "--partition-tags", "--odd-records", "--contig-tag", "XC"]
DEVICES = ("0,0", "0,0,0", "0,0,0,0,0")


def pt(*tags):
    return [a for t in tags for a in ("--partition-tag", t)]


CASES = [
    ("rg_hp_cpg", pt("RG", "HP") + ["--cpg", "--ref", "@FA"], True),
    ("xf_prefix", pt("XF") + ["--prefix", "f", "-i", "30011"], False),
    ("hp_traditional", pt("HP") + ["--preset", "traditional", "--ref", "@FA"], True),
    ("hp_cpg_combine", pt("HP") + ["--cpg", "--combine-strands", "--ref", "@FA"], False),
    ("five_tags", pt("XX", "HP", "YY", "XF", "RG") + ["-i", "50021"], False),
    ("include_bed", pt("HP") + ["--include-bed", "@BED"], False),
    ("region", pt("RG") + ["--region", "c1:100000-350000", "-i", "40000"], False),
    ("max_depth", pt("HP") + ["--max-depth", "6"], False),
    ("small_chunks", pt("RG") + ["--gpu-chunk-bp", "50000"], False),
]


@pytest.fixture(scope="module")
def genome(synth_exe, tmp_path_factory):
    d = tmp_path_factory.mktemp("pgen")
    prefix, _ = synth(synth_exe, d, "g", *GENOME)
    with open(prefix + ".bed", "w") as f:
        f.write("c1\t1000\t60000\n" "c1\t200000\t230000\n" "c2\t0\t160000\n" "c4\t120000\t121000\n")
    return prefix


def expand(flags, prefix):
    return [prefix + ".fa" if f == "@FA" else prefix + ".bed" if f == "@BED" else f for f in flags]


def run_dir(flags, bam, out):
    rc, _ = run_product(flags, bam, out)
    assert rc == 0, (flags, out)
    return read_dir(out)


@pytest.mark.parametrize("name,flags,with_oracle", CASES, ids=[c[0] for c in CASES])
def test_gpu_partition_devices_equal_single(name, flags, with_oracle, genome, native_lib, oracle_exe, tmp_path):
    flags = expand(flags, genome)
    one = run_dir(flags, genome + ".bam", str(tmp_path / "one"))
    assert len(one) >= 2 and sum(len(t) for t in one.values()) > 10000
    if with_oracle:
        oflags = [f for i, f in enumerate(flags) if f != "--gpu-chunk-bp" and (i == 0 or flags[i - 1] != "--gpu-chunk-bp")]
        subprocess.check_call([oracle_exe, "pileup", "-t", "8"] + oflags + [genome + ".bam", str(tmp_path / "oracle")], stderr=subprocess.DEVNULL)
        assert read_dir(str(tmp_path / "oracle")) == one
    for devs in DEVICES:
        got = run_dir(flags + ["--devices", devs], genome + ".bam", str(tmp_path / ("d%d" % len(devs))))
        assert sorted(got) == sorted(one)
        for f in one:
            assert got[f] == one[f], (devs, f)


def test_gpu_partition_uneven_shards(genome, native_lib, oracle_exe, tmp_path):
    import modkit_b200
    bam = genome + ".bam"
    # one interval per contig, five ranks: some rank has no interval and every contig (= XC value) lies in one shard
    plan = modkit_b200.shard_plan(bam, 1000000, 5)
    ranks_of = {}
    for r, tid, _, _ in plan:
        ranks_of.setdefault(tid, set()).add(r)
    assert len({r for r, _, _, _ in plan}) < 5
    assert all(len(v) == 1 for v in ranks_of.values())
    flags = pt("XC", "HP") + ["-i", "1000000"]
    one = run_dir(flags, bam, str(tmp_path / "one"))
    subprocess.check_call([oracle_exe, "pileup", "-t", "8"] + flags + [bam, str(tmp_path / "oracle")], stderr=subprocess.DEVNULL)
    assert read_dir(str(tmp_path / "oracle")) == one
    assert any(f.startswith("c3_") for f in one)
    assert run_dir(flags + ["--devices", "0,0,0,0,0"], bam, str(tmp_path / "d5")) == one
    # the default grid on three ranks: c3 (the smallest contig) is one rank's only, so its XC values are written by one rank
    plan = modkit_b200.shard_plan(bam, 100000, 3)
    assert len({r for r, tid, _, _ in plan if tid == 2}) == 1
    flags = pt("XC")
    one = run_dir(flags, bam, str(tmp_path / "one3"))
    assert sorted(one) == ["c1.bed", "c2.bed", "c3.bed", "c4.bed"]
    assert run_dir(flags + ["--devices", "0,0,0"], bam, str(tmp_path / "d3")) == one
    # a region inside one interval: only rank 0 has rows
    flags = pt("HP", "XC") + ["--region", "c2:20000-70000"]
    one = run_dir(flags, bam, str(tmp_path / "oner"))
    assert run_dir(flags + ["--devices", "0,0,0,0,0"], bam, str(tmp_path / "dr")) == one


def test_gpu_partition_stale_directory(genome, native_lib, tmp_path):
    bam = genome + ".bam"
    flags = pt("HP")
    one = run_dir(flags, bam, str(tmp_path / "one"))
    assert "1.bed" in one
    out = tmp_path / "stale"
    out.mkdir()
    (out / "1.bed").write_text(one["1.bed"] * 2 + "stale tail\n")
    (out / "unrelated.txt").write_text("keep me\n")
    (out / "2_x.bed").write_text("a partition this run does not make\n")
    rc, _ = run_product(flags + ["--devices", "0,0,0"], bam, str(out))
    assert rc == 0
    got = read_dir(str(out))
    assert got.pop("unrelated.txt") == "keep me\n" and got.pop("2_x.bed") == "a partition this run does not make\n"
    assert got == one


def test_gpu_partition_sharded_errors_are_clean(genome, native_lib, tmp_path):
    rc, _ = run_product(pt("HP") + ["--filter-threshold", "Q:0.5", "--devices", "0,0"], genome + ".bam", str(tmp_path / "e"))
    assert rc == 1


def value_text(ty, raw):
    import modkit_b200
    c = chr(ty)
    if c in "ZH":
        return raw.decode()
    if c == "A":
        return raw.decode()
    if c == "f":
        return modkit_b200.f32_display(struct.unpack("<f", raw)[0])
    return str(struct.unpack("<" + {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I"}[c], raw)[0])


def key_of(types, lens, offs, values, i):
    parts = [value_text(types[i, t], values[offs[i, t]:offs[i, t] + lens[i, t]]) if types[i, t] else None for t in range(types.shape[1])]
    return None if all(p is None for p in parts) else "_".join("missing" if p is None else p for p in parts)


def test_gpu_tag_values_equal_host(native_lib, synth_exe, tmp_path):
    """mkp_bam_tag_values against the host's aux reader, record by record: long Z and H values, A/C/i/f scalars, B arrays and absent
    tags count as missing."""
    import modkit_b200 as mk
    long_prefix, _ = synth(synth_exe, tmp_path, "lt", "--contig", "syn1:150000", "--coverage", "10", "--mods", "m", "--seed", "61", "--long-tags")
    short_prefix, _ = synth(synth_exe, tmp_path, "st", "--contig", "syn1:150000", "--coverage", "10", "--mods", "hm", "--seed", "62", "--partition-tags", "--odd-records")
    seen = set()
    for path in (long_prefix + ".bam", short_prefix + ".bam"):
        host = mk.Bam(path, threads=2)
        c = mk.Context(0)
        dev = mk.Bam(path, ctx=c)
        n = host.n_records(0)
        assert n > 0
        ids = np.arange(n, dtype=np.uint32)
        for tags in (["RG", "XH"], ["XH", "ML", "RG", "HP"], ["XX"], ["HP", "XF", "MM", "YY"]):
            types, lens, offs, values = c.bam_tag_values(ids, tags)
            assert (offs.ravel()[1:] == np.cumsum(lens.ravel())[:-1]).all() and len(values) == int(lens.sum())
            for i in range(n):
                assert key_of(types, lens, offs, values, i) == host.partition_key(0, i, tags), (path, tags, i)
            seen |= {int(x) for x in lens.ravel()} | {chr(x) for x in types.ravel() if x}
            if "ML" in tags:
                assert (types[:, tags.index("ML")] == 0).all()                # B arrays are not stringable
        # the sharded pileup partitions these records through the same values
        dev.close(); host.close(); c.close()
    assert {254, 255, 256, 1000, 70000} <= seen and {"Z", "H", "C", "i", "f"} <= seen


def test_gpu_long_partition_values_run_alike(native_lib, oracle_exe, synth_exe, tmp_path, capfd):
    """A partition key longer than a file name can be fails the same way on every front end: device ingest (no more 253-byte
    limit), host ingest, three shards and the oracle; a partition over a short tag of the same reads gives the same directories."""
    prefix, _ = synth(synth_exe, tmp_path, "lt", "--contig", "syn1:150000", "--contig", "syn2:80000", "--coverage", "10", "--mods", "m", "--seed", "63",
                      "--long-tags", "--contig-tag", "XC")
    bam = prefix + ".bam"
    for k, extra in enumerate(([], ["--host-ingest"], ["--devices", "0,0,0"])):
        rc, _ = run_product(pt("RG") + extra, bam, str(tmp_path / ("long%d" % k)))
        assert rc == 1
        err = capfd.readouterr().err
        assert "longer than 253" not in err and "failed to make output file" in err, err[-500:]
    assert subprocess.run([oracle_exe, "pileup", "--partition-tag", "RG", bam, str(tmp_path / "olong")], capture_output=True).returncode != 0
    one = run_dir(pt("XC", "YY"), bam, str(tmp_path / "one"))
    subprocess.check_call([oracle_exe, "pileup", "-t", "8"] + pt("XC", "YY") + [bam, str(tmp_path / "oracle")], stderr=subprocess.DEVNULL)
    assert read_dir(str(tmp_path / "oracle")) == one
    assert run_dir(pt("XC", "YY") + ["--host-ingest"], bam, str(tmp_path / "host")) == one
    assert run_dir(pt("XC", "YY") + ["--devices", "0,0,0"], bam, str(tmp_path / "d3")) == one


def test_gpu_partition_torchrun_nccl(genome, native_lib, tmp_path):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    flags = pt("HP")
    one = run_dir(flags, genome + ".bam", str(tmp_path / "one"))
    for world in sorted({2, min(n, 4)}):
        out = str(tmp_path / ("w%d" % world))
        p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                            "--master-port", str(29600 + world), os.path.join(ROOT, "tests", "sharded_worker.py")] + flags + [genome + ".bam", out],
                           capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        assert read_dir(out) == one
