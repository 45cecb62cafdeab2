#!/usr/bin/env python
"""Where the warps of the fast k_resolve spend their cycles: per-phase shares of the clock64() counters of a measurement build.

    tools/build_variant.sh rclk WORK -DMKP_RESOLVE_CLOCKS=1
    MODKIT_B200_LIB=$PWD/modkit_b200/_build/variants/rclk.so python tools/resolve_phases.py [--len 64444167] [--coverage 40]
        [--steps 5] [--warmup 3] [--out FILE]

Same chunk, seed and pass as tools/pass_profile.py (one 64.4 Mb chunk of the bench workload, `--cpg --combine-strands` focus,
numeric mode 2 collapsing `h`, C threshold 0.6). After --warmup passes the counters are zeroed, --steps passes run, and the
counters are read back (mkp_debug_resolve_clocks, present only in builds with MKP_RESOLVE_CLOCKS). Each warp of
k_resolve<MODE_PILEUP, true> sums, over the reads it takes from the queue, the SM cycles between phase boundaries; a round of 32
list entries is split at the slowest lane's end of the call. The shares are of all warps' summed cycles, so they weigh latency
the warp waits on and issue alike. Prints the card's name, power limit and max SM clock, then one line per phase."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pass_profile import SEED, card  # noqa: E402

PHASES = ["queue + header + lists", "CIGAR prefix", "query -> op table", "per-entry resolve", "projection + emit", "commit"]


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
    import modkit_b200
    lib = modkit_b200.load_library()
    if not hasattr(lib, "mkp_debug_resolve_clocks"):
        sys.exit("%s has no k_resolve phase counters: build it with -DMKP_RESOLVE_CLOCKS=1 and pass it in MODKIT_B200_LIB" % modkit_b200.library_path())
    lib.mkp_debug_resolve_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
    n_ctr = 8
    buf = (C.c_ulonglong * n_ctr)()
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
        if lib.mkp_debug_resolve_clocks(buf, n_ctr, 1) != n_ctr:
            sys.exit("mkp_debug_resolve_clocks failed")
        resolve_ms = 0.0
        for _ in range(a.steps):
            resolve_ms += float(ctx.pileup_resident().kernel_ms[1])
        if lib.mkp_debug_resolve_clocks(buf, n_ctr, 0) != n_ctr:
            sys.exit("mkp_debug_resolve_clocks failed")
        bam.close()
        ctx.close()
    v = np.array(list(buf), dtype=np.float64)
    cyc, reads, entries = v[:6], v[6], v[7]
    total = cyc.sum()
    lines = ["card: %s" % card(),
             "library: %s" % os.path.basename(modkit_b200.library_path()),
             "chunk: %d bp at %gx, %d reads; %d passes after %d warm-up passes; resolve stage %.3f ms per pass (CUDA events, counting build)"
             % (a.len, a.coverage, n_reads, a.steps, a.warmup, resolve_ms / a.steps),
             "reads resolved by the fast kernel per pass: %d; list entries per read: %.1f; warp cycles per read: %.0f"
             % (reads / a.steps, entries / max(reads, 1), total / max(reads, 1)),
             "%-24s %16s %14s %7s" % ("phase", "warp cycles", "per read", "share")]
    for name, c in zip(PHASES, cyc):
        lines.append("%-24s %16.0f %14.0f %6.1f%%" % (name, c, c / max(reads, 1), 100.0 * c / total if total else 0.0))
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
