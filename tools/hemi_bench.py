#!/usr/bin/env python
"""Timing of the resident `pileup-hemi` pass beside the resident `--cpg --combine-strands` pileup pass, on the same chunk.

    python tools/hemi_bench.py [--len 16111041] [--coverage 40] [--steps 7] [--warmup 2] [--out profiles/h100_hemi_bench.json]

Input: one seeded synthetic duplex contig (tools/synth_modbam --duplex --mods hm: C+h?/C+m? and G-h?/G-m? lists, 6% of the reads
without usable tags) of --len bp at --coverage, generated in a temporary directory. The default, 16,111,041 bp at 40x, is a
quarter of chr20: 1/16 of the bench.py genome at its coverage. The BAM is inflated and sliced on the GPU; the whole contig is
one resident chunk, its CpGs on the 100 kb interval grid are the focus, the thresholds are fixed (C: 0.8).

Each step times both passes, alternating: mkp_pileup_resident with the combine-strands focus bitmaps (the device pass of
`pileup --cpg --combine-strands`; the host's strand combining is not included) and mkp_hemi_resident with the + strand CpGs
(partner offset +1). A pass returns after a stream synchronise, so the host clock around it is the pass time; the CUDA-event
total the pass reports (stats.kernel_ms[7]) is recorded beside it. Median over --steps after --warmup passes of each. The
card's name and power limit are read in the same run. Prints one JSON line and writes it to --out when given."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    first = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    parts = [p.strip() for p in first.split(",")]
    return {"gpu": parts[0] if parts else "", "power_limit": parts[1] if len(parts) > 1 else "", "max_sm_clock": parts[2] if len(parts) > 2 else ""}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--len", type=int, default=16_111_041)
    ap.add_argument("--coverage", type=float, default=40)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=20261015)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if a.steps < 5:
        sys.exit("--steps must be >= 5 (the median of at least five passes)")
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement runs on the GPU only")
    import modkit_b200
    synth = os.path.join(ROOT, "tools", "_build", "synth_modbam")
    if not os.path.exists(synth):
        os.makedirs(os.path.dirname(synth), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(ROOT, "tools", "synth_modbam.cpp"), "-o", synth, "-lz"])
    with tempfile.TemporaryDirectory() as td:
        prefix = os.path.join(td, "duplex")
        t0 = time.perf_counter()
        info = json.loads(subprocess.run([synth, "--out", prefix, "--contig", "syn1:%d" % a.len, "--coverage", str(a.coverage), "--mods", "hm",
                                          "--duplex", "--seed", str(a.seed), "--threads", str(os.cpu_count() or 8)],
                                         capture_output=True, text=True, check=True).stdout)
        gen_s = time.perf_counter() - t0
        ctx = modkit_b200.Context(0)
        bam = modkit_b200.Bam(prefix + ".bam", ctx=ctx)
        ctx.set_params(modkit_b200.make_params(base_thresholds={"C": 0.8}))
        fpos, fneg = modkit_b200.motif_focus(prefix + ".fa", "syn1", 0, a.len, 100000, "CG:0", True)
        n_reads = bam.device_chunk(0, 0, a.len, focus=(fpos, fneg))
        starts = list(range(0, a.len, 100000))
        pile = lambda: ctx.pileup_resident()                     # noqa: E731
        hemi = lambda: ctx.hemi_resident(starts, 1)              # noqa: E731
        for _ in range(a.warmup):
            pile(); hemi()
        wall = {"pileup": [], "hemi": []}
        ev = {"pileup": [], "hemi": []}
        rows = {}
        for _ in range(a.steps):
            for name, fn in (("pileup", pile), ("hemi", hemi)):
                t = time.perf_counter()
                st = fn()
                wall[name].append((time.perf_counter() - t) * 1e3)
                ev[name].append(float(st.kernel_ms[7]))
                rows[name] = int(st.n_rows)
        focus_pos = int(sum(bin(int(w)).count("1") for w in fpos))
        rec = {"what": "resident passes over one chunk: pileup-hemi (--cpg) vs pileup --cpg --combine-strands (device pass)",
               "contig_bp": a.len, "coverage": a.coverage, "reads": n_reads, "read_bases": info["read_bases"], "plus_strand_cpgs": focus_pos,
               "steps": a.steps, "warmup": a.warmup, "generate_s": round(gen_s, 2)}
        for name in ("hemi", "pileup"):
            ms = statistics.median(wall[name])
            rec[name] = {"ms_median": round(ms, 3), "ms_all": [round(x, 3) for x in wall[name]], "event_ms_median": round(statistics.median(ev[name]), 3),
                         "positions_per_s": round(a.len / (ms / 1e3)), "cpgs_per_s": round(focus_pos / (ms / 1e3)), "rows": rows[name]}
        rec["hemi_over_pileup"] = round(rec["hemi"]["ms_median"] / rec["pileup"]["ms_median"], 3)
        rec.update(card())
        rec["torch_device_name"] = torch.cuda.get_device_name(0)
        line = json.dumps(rec)
        print(line)
        if a.out:
            with open(a.out, "w") as fh:
                fh.write(line + "\n")
        bam.close()
        ctx.close()


if __name__ == "__main__":
    main()
