#!/usr/bin/env python
"""Per-kernel time of the resident pileup pass, from torch.profiler (CUDA activities).

    python tools/pass_profile.py [--len 64444167] [--coverage 40] [--steps 5] [--warmup 3] [--out FILE]

Input: one chunk of the bench.py workload: a seeded synthetic contig of --len bp (default: chr20, one quarter of the bench
genome) at --coverage, with the bench's generator flags (`--mods hm --level 1`, same seed), generated in a temporary directory.
The pass is the bench's: `--cpg --combine-strands` focus bitmaps on the 100 kb interval grid, numeric mode 2 collapsing `h`,
a fixed C threshold of 0.6. After --warmup passes, --steps passes run under the profiler. Prints one line per kernel (total
and per-pass ms, launches per pass, share of the kernel time), the card's name, power limit and max SM clock, and the pass's
own CUDA-event stage times (stats.kernel_ms). With --out, the same text is written there."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = 20260924          # bench.py's generator seed


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--len", type=int, default=64_444_167)
    ap.add_argument("--coverage", type=float, default=40)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement runs on the GPU only")
    from torch.profiler import ProfilerActivity, profile
    import modkit_b200
    synth = os.path.join(ROOT, "tools", "_build", "synth_modbam")
    if not os.path.exists(synth):
        os.makedirs(os.path.dirname(synth), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(ROOT, "tools", "synth_modbam.cpp"), "-o", synth, "-lz"])
    with tempfile.TemporaryDirectory() as td:
        prefix = os.path.join(td, "w")
        subprocess.run([synth, "--out", prefix, "--contig", "syn1:%d" % a.len, "--coverage", str(a.coverage), "--mods", "hm", "--seed", str(SEED),
                        "--level", "1", "--threads", str(min(96, os.cpu_count() or 8))], check=True, capture_output=True)
        ctx = modkit_b200.Context(0)
        bam = modkit_b200.Bam(prefix + ".bam", ctx=ctx)
        fpos, fneg = modkit_b200.motif_focus(prefix + ".fa", "syn1", 0, a.len, 100000, "CG:0", True)
        ctx.set_params(modkit_b200.make_params(base_thresholds={"C": 0.6}, numeric_mode=2, collapse_code="h"))
        n_reads = bam.device_chunk(0, 0, a.len, focus=(fpos, fneg))
        for _ in range(a.warmup):
            ctx.pileup_resident()
        torch.cuda.synchronize()
        stage = np.zeros(8)
        l0 = ctx.kernel_launches
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                st = ctx.pileup_resident()
                stage += np.array(list(st.kernel_ms))
            torch.cuda.synchronize()
        launches = (ctx.kernel_launches - l0) / a.steps
        stage /= a.steps
        n_rows = int(st.n_rows)
        bam.close()
        ctx.close()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or e.device_time <= 0:
            continue
        t, c = per.get(e.name, (0.0, 0))
        per[e.name] = (t + e.device_time / 1e3, c + 1)          # device_time: us
    total = sum(t for t, _ in per.values())
    lines = ["card: %s" % card(),
             "chunk: %d bp at %gx, %d reads, %d rows; %d profiled passes after %d warm-up passes; %.1f launches per pass (library count)"
             % (a.len, a.coverage, n_reads, n_rows, a.steps, a.warmup, launches),
             "%-60s %10s %10s %8s %7s" % ("kernel / activity", "total ms", "ms/pass", "n/pass", "share")]
    for name, (t, c) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        lines.append("%-60s %10.3f %10.3f %8.2f %6.1f%%" % (name[:60], t, t / a.steps, c / a.steps, 100.0 * t / total if total else 0.0))
    lines.append("%-60s %10.3f %10.3f" % ("sum of device activity", total, total / a.steps))
    names = ["parse", "resolve", "rank", "count_calls", "counters", "rows", "host", "total"]
    lines.append("stats.kernel_ms per pass (CUDA events, profiler on): " + json.dumps({n: round(float(x), 3) for n, x in zip(names, stage)}))
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
