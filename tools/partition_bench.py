#!/usr/bin/env python
"""Timing of a haplotype-partitioned pileup, file -> directory: `modkit pileup --partition-tag HP --cpg --combine-strands --ref`
on one device against `--devices 0,...,N-1` on the N GPUs present.

    python tools/partition_bench.py [--len 64444167] [--coverage 40] [--rounds 3] [--out profiles/h100_partition_bench.json]

Input: one seeded synthetic contig (tools/synth_modbam --partition-tags --mods hm: RG:Z on 90% of the reads, HP as C (1, 2) or
i (3) on 80%, XF:f on some) of --len bp at --coverage (the default is chr20 at bench.py's coverage), generated in a temporary
directory. Each round runs the one-device arm and then the N-device arm, in process; a run's time is the host clock around it,
output files written. The median of --rounds alternating rounds is reported, and the two directories are checked to be equal.
With one GPU only the one-device arm is timed: scaling is then not measured, and the result says so.

The tag bytes copied to the host by the partition step are counted, not measured, from the raw values of every record (all
admitted; each record once; a read in two chunks is fetched in each): mkp_bam_tags copies MKP_TAG_CELL = 256 bytes per (record, tag),
mkp_bam_tag_values copies 9 bytes per (record, tag) (type, length, offset) plus the value bytes. The card's name and power
limit are read in the same run. Prints one JSON line and writes it to --out when given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

COVERAGE = 40          # bench.py's COVERAGE


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    first = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    parts = [p.strip() for p in first.split(",")]
    return {"gpu": parts[0] if parts else "", "power_limit": parts[1] if len(parts) > 1 else "", "max_sm_clock": parts[2] if len(parts) > 2 else ""}


def read_dir(path):
    return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}


def tag_bytes(modkit_b200, bam_path, tags):
    """(records, bytes copied by the 256-byte cells, bytes copied by the values) for every record of the file, each once (the
    generator's reads are all mapped primary alignments, so every record is one the pileup admits)."""
    import numpy as np
    ctx = modkit_b200.Context(0)
    bam = modkit_b200.Bam(bam_path, ctx=ctx)
    n = bam.total_records
    after = 0
    for k in range(0, n, 1 << 20):
        types, lens, offs, values = ctx.bam_tag_values(np.arange(k, min(n, k + (1 << 20)), dtype=np.uint32), tags)
        after += types.size * 9 + len(values)
    bam.close()
    ctx.close()
    return n, n * len(tags) * 256, after


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--len", type=int, default=64_444_167)
    ap.add_argument("--coverage", type=float, default=COVERAGE)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=20261018)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement runs on the GPU only")
    import modkit_b200
    n_gpu = torch.cuda.device_count()
    synth = os.path.join(ROOT, "tools", "_build", "synth_modbam")
    if not os.path.exists(synth):
        os.makedirs(os.path.dirname(synth), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(ROOT, "tools", "synth_modbam.cpp"), "-o", synth, "-lz"])
    base = "/dev/shm" if os.path.isdir("/dev/shm") else None
    with tempfile.TemporaryDirectory(dir=base) as td:
        prefix = os.path.join(td, "hp")
        t0 = time.perf_counter()
        info = json.loads(subprocess.run([synth, "--out", prefix, "--contig", "chr20:%d" % a.len, "--coverage", str(a.coverage), "--mods", "hm",
                                          "--partition-tags", "--seed", str(a.seed), "--threads", str(min(64, os.cpu_count() or 8))],
                                         capture_output=True, text=True, check=True).stdout)
        gen_s = time.perf_counter() - t0
        flags = ["--partition-tag", "HP", "--cpg", "--combine-strands", "--ref", prefix + ".fa", "--quiet"]
        arms = [("one_device", [])]
        if n_gpu > 1:
            arms.append(("devices_%d" % n_gpu, ["--devices", ",".join(str(d) for d in range(n_gpu))]))
        secs = {name: [] for name, _ in arms}
        dirs = {}
        for r in range(a.rounds):
            for name, extra in arms:
                out = os.path.join(td, "%s_%d" % (name, r))
                t = time.perf_counter()
                rc = modkit_b200.pileup_main(flags + extra + [prefix + ".bam", out])
                secs[name].append(time.perf_counter() - t)
                if rc != 0:
                    sys.exit("pileup failed (%s, exit %d)" % (name, rc))
                dirs[name] = out
        files = read_dir(dirs["one_device"])
        same = all(read_dir(d) == files for d in dirs.values())
        n_adm, before, after = tag_bytes(modkit_b200, prefix + ".bam", ["HP"])
        rec = {"what": "modkit pileup --partition-tag HP --cpg --combine-strands, file -> directory, one device vs --devices over all GPUs",
               "contig_bp": a.len, "coverage": a.coverage, "reads": info["reads"], "bam_bytes": info["bam_bytes"], "generate_s": round(gen_s, 2),
               "gpus": n_gpu, "rounds": a.rounds, "files": sorted(files), "output_bytes": sum(len(v) for v in files.values()), "directories_equal": same}
        for name, _ in arms:
            rec[name] = {"s_median": round(statistics.median(secs[name]), 3), "s_all": [round(x, 3) for x in secs[name]]}
        if n_gpu > 1:
            rec["speedup"] = round(rec["one_device"]["s_median"] / rec["devices_%d" % n_gpu]["s_median"], 3)
        else:
            rec["scaling"] = "not measured: one GPU"
        rec["tag_bytes_to_host"] = {"counted_not_measured": True, "records": n_adm, "n_tags": 1,
                                    "cells_256_per_tag": before, "values": after}
        rec.update(card())
        line = json.dumps(rec)
        print(line)
        if a.out:
            with open(a.out, "w") as fh:
                fh.write(line + "\n")
        if not same:
            sys.exit("the directories differ")


if __name__ == "__main__":
    main()
