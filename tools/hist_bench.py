#!/usr/bin/env python
"""Cost of `sample-probs --hist` on the GPU.

    python tools/hist_bench.py [--len 16000000] [--coverage 30] [--rounds 3] [--out profiles/h100_sample_probs_hist.log]

Input: one seeded synthetic contig (tools/synth_modbam --mods hma) of --len bp at --coverage, generated in a temporary directory.

Two measurements, each alternating the two variants round by round, median over --rounds after one warm-up of each:
  * end to end: `modkit sample-probs --no-sampling` with the table on stdout, and with `-o DIR --hist` (which adds a second
    decode pass over the sampled reads and writes the four files). Host clock around the whole command.
  * the decode pass alone, on the contig as one resident chunk: mkp_sample_histogram_wide (the sampling decode) against
    mkp_sample_mod_histogram (the same decode with the per-(state, qual) counters in global memory). Each call ends in a stream
    synchronise, so the host clock around it is its device time plus one small copy back.
The card's name and power limit are read in the same run. Prints the log and writes it to --out when given."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--len", type=int, default=16_000_000)
    ap.add_argument("--coverage", type=float, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--decode-reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=20261016)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import modkit_b200
    modkit = os.path.join(ROOT, "modkit_b200", "_build", "modkit")
    synth = os.path.join(ROOT, "tools", "_build", "synth_modbam")
    if not os.path.exists(synth):
        os.makedirs(os.path.dirname(synth), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(ROOT, "tools", "synth_modbam.cpp"), "-o", synth, "-lz"])
    lines = ["card: " + card()]
    with tempfile.TemporaryDirectory() as td:
        prefix = os.path.join(td, "g")
        info = json.loads(subprocess.run([synth, "--out", prefix, "--contig", "syn1:%d" % a.len, "--coverage", str(a.coverage), "--mods", "hma",
                                          "--seed", str(a.seed), "--threads", str(os.cpu_count() or 8)], capture_output=True, text=True, check=True).stdout)
        bam = prefix + ".bam"
        lines.append("input: syn1 %d bp at %sx, %s" % (a.len, a.coverage, json.dumps(info)))
        variants = {"stdout": [], "hist": []}

        def run(v, k):
            args = [modkit, "sample-probs", "--no-sampling", "-t", "8", bam]
            if v == "hist":
                args += ["-o", os.path.join(td, "out%d" % k), "--hist"]
            t0 = time.perf_counter()
            p = subprocess.run(args, capture_output=True, text=True)
            dt = time.perf_counter() - t0
            if p.returncode != 0:
                sys.exit("sample-probs failed: " + p.stderr)
            return dt
        for v in variants:
            run(v, 99)
        for k in range(a.rounds):
            for v in variants:
                variants[v].append(run(v, k))
        for v, ts in variants.items():
            lines.append("end to end %-6s: median %.3f s  runs %s" % (v, statistics.median(ts), " ".join("%.3f" % t for t in ts)))
        med = {v: statistics.median(ts) for v, ts in variants.items()}
        lines.append("end to end: --hist -o adds %.1f %%" % (100.0 * (med["hist"] / med["stdout"] - 1.0)))
        # the decode pass alone
        b = modkit_b200.Bam(bam, threads=8)
        ctx = modkit_b200.Context(0)
        ctx.set_params(modkit_b200.make_params(force_allow_implicit=True))
        ctx.upload(b.pack(0, 0, b.refs[0][1]))
        calls = {"wide": lambda: ctx.sample_histogram(include_unaligned=True, wide=True),
                 "mod_hist": lambda: ctx.sample_mod_histogram(include_unaligned=True)}
        hw, _, _ = calls["wide"]()
        hq, _ = calls["mod_hist"]()
        assert int(hw.sum()) == int(hq.sum()), (int(hw.sum()), int(hq.sum()))
        lines.append("decode chunk: %d reads, %d arg-max values" % (b.n_records(0), int(hq.sum())))
        times = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, fn in calls.items():
                t0 = time.perf_counter()
                for _ in range(a.decode_reps):
                    fn()
                times[k].append((time.perf_counter() - t0) / a.decode_reps * 1e3)
        for k, ts in times.items():
            lines.append("decode %-8s: median %.3f ms  rounds %s" % (k, statistics.median(ts), " ".join("%.3f" % t for t in ts)))
        lines.append("decode: the qhist counters add %.1f %%" % (100.0 * (statistics.median(times["mod_hist"]) / statistics.median(times["wide"]) - 1.0)))
        ctx.close()
        b.close()
    text = "\n".join(lines) + "\n"
    print(text, end="")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(text)


if __name__ == "__main__":
    main()
