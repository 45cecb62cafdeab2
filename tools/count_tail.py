#!/usr/bin/env python
"""The tail of k_count_bases: when its work items are dequeued and finished, from the item log of a measurement build.

    tools/build_variant.sh cclk WORK -DMKP_COUNT_CLOCKS=1
    MODKIT_B200_LIB=$PWD/modkit_b200/_build/variants/cclk.so python tools/count_tail.py [--item-bp 16384,...] [--len 64444167]
        [--coverage 40] [--steps 5] [--warmup 3] [--out FILE]

Same chunk, seed and pass as tools/pass_profile.py (one 64.4 Mb chunk of the bench workload, `--cpg --combine-strands` focus,
numeric mode 2 collapsing `h`, C threshold 0.6). For every window size of --item-bp (MKP_COUNT_ITEM_BP, read when the chunk is
uploaded; 1073741824 = one item per read, the queue the kernel had before it took windows) the chunk is uploaded again, --warmup
passes run, then --steps passes each log every item k_count_bases takes: its SM and %globaltimer at dequeue and at the warp's next
dequeue (mkp_debug_count_clocks, present only in builds with MKP_COUNT_CLOCKS). Per pass:

  span       first dequeue -> last finish (the kernel, less its launch and the exit of the last warp)
  tail       last dequeue -> last finish
  idle       warp-slot time left idle after the last dequeue, as a share of slots x span; slots = the most items in flight
  counters   the pass's counting stage (CUDA events: k_count_bases, with k_count_calls beside it)

Medians over the passes are printed, then the ten longest items of the last pass. Prints the card's name, power limit and max SM
clock first."""
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

REC = [("t0", "<u8"), ("t1", "<u8"), ("sm", "<u4"), ("read", "<u4"), ("r_lo", "<u4"), ("r_hi", "<u4")]   # CountClk


def tail_stats(log, np):
    log = log[log["t1"] != 0]
    t0, t1 = log["t0"].astype(np.int64), log["t1"].astype(np.int64)
    T0, T1, Tq = int(t0.min()), int(t1.max()), int(t0.max())
    ev = np.concatenate([np.stack([t0, np.ones_like(t0)], 1), np.stack([t1, -np.ones_like(t1)], 1)])
    ev = ev[np.lexsort((ev[:, 1], ev[:, 0]))]            # finishes before starts at equal times
    slots = int(np.cumsum(ev[:, 1]).max())
    busy_after = np.clip(t1 - np.maximum(t0, Tq), 0, None).sum()
    idle_after = slots * (T1 - Tq) - busy_after
    return {"items": len(log), "span_ms": (T1 - T0) / 1e6, "tail_ms": (T1 - Tq) / 1e6, "slots": slots,
            "idle_share": idle_after / (slots * (T1 - T0)), "T0": T0, "log": log}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--item-bp", default="1073741824,8192,16384,32768")
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
    if not hasattr(lib, "mkp_debug_count_clocks"):
        sys.exit("%s has no k_count_bases item log: build it with -DMKP_COUNT_CLOCKS=1 and pass it in MODKIT_B200_LIB" % modkit_b200.library_path())
    lib.mkp_debug_count_clocks.argtypes = [C.c_void_p, C.c_uint32]
    cap = 1 << 20
    synth = os.path.join(ROOT, "tools", "_build", "synth_modbam")
    if not os.path.exists(synth):
        os.makedirs(os.path.dirname(synth), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", os.path.join(ROOT, "tools", "synth_modbam.cpp"), "-o", synth, "-lz"])
    lines = ["card: %s" % card(), "library: %s" % os.path.basename(modkit_b200.library_path())]
    with tempfile.TemporaryDirectory() as td:
        prefix = os.path.join(td, "w")
        subprocess.run([synth, "--out", prefix, "--contig", "syn1:%d" % a.len, "--coverage", str(a.coverage), "--mods", "hm", "--seed", str(SEED),
                        "--level", "1", "--threads", str(min(96, os.cpu_count() or 8))], check=True, capture_output=True)
        ctx = modkit_b200.Context(0)
        bam = modkit_b200.Bam(prefix + ".bam", ctx=ctx)
        fpos, fneg = modkit_b200.motif_focus(prefix + ".fa", "syn1", 0, a.len, 100000, "CG:0", True)
        ctx.set_params(modkit_b200.make_params(base_thresholds={"C": 0.6}, numeric_mode=2, collapse_code="h"))
        lines.append("chunk: %d bp at %gx; %d passes after %d warm-up passes per window size; medians over the passes" % (a.len, a.coverage, a.steps, a.warmup))
        lines.append("%12s %8s %9s %9s %9s %7s %10s" % ("item bp", "items", "span ms", "tail ms", "idle", "slots", "counters"))
        for bp in [int(x) for x in a.item_bp.split(",")]:
            os.environ["MKP_COUNT_ITEM_BP"] = str(bp)
            n_reads = bam.device_chunk(0, 0, a.len, focus=(fpos, fneg))
            for _ in range(a.warmup):
                ctx.pileup_resident()
            runs, stage = [], []
            for _ in range(a.steps):
                if lib.mkp_debug_count_clocks(None, cap) != 0:
                    sys.exit("mkp_debug_count_clocks failed")
                stage.append(float(ctx.pileup_resident().kernel_ms[4]))
                buf = np.zeros(cap, dtype=REC)
                if lib.mkp_debug_count_clocks(buf.ctypes.data, cap) != 0:
                    sys.exit("mkp_debug_count_clocks failed")
                runs.append(tail_stats(buf, np))
            med = {k: float(np.median([r[k] for r in runs])) for k in ("items", "span_ms", "tail_ms", "idle_share", "slots")}
            lines.append("%12d %8d %9.3f %9.3f %8.2f%% %7d %10.3f" % (bp, med["items"], med["span_ms"], med["tail_ms"], 100 * med["idle_share"],
                                                                     med["slots"], float(np.median(stage))))
            last = runs[-1]
            log = last["log"]
            dur = (log["t1"] - log["t0"]).astype(np.int64)
            top = np.argsort(-dur)[:10]
            lines.append("  ten longest items of the last pass (%d reads): us, dequeued at us, SM, read, [r_lo, r_hi) length" % n_reads)
            for k in top:
                lines.append("    %8.1f %9.1f %4d %8d %8d" % (dur[k] / 1e3, (int(log["t0"][k]) - last["T0"]) / 1e3, log["sm"][k], log["read"][k],
                                                          int(log["r_hi"][k]) - int(log["r_lo"][k])))
        os.environ.pop("MKP_COUNT_ITEM_BP", None)
        bam.close()
        ctx.close()
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
