#!/usr/bin/env python
"""Regenerates the `pileup-hemi` fixtures under tests/golden/generated/ from the reference's own fixtures. The outputs are
committed, so the tests need no checkout of the reference.

    python tests/golden/make_duplex_fixtures.py <path to a nanoporetech/modkit v0.4.4 checkout>

The reference's tests (tests/test_pileup_hemi.rs) use tests/resources/duplex_modcalls_sort.bam (2.1 MB) and GRCh38_chr20.fa
(65 MB); this keeps the window those tests look at, each file under 1 MB:
duplex_window.bam(.bai)   = the duplex reads that overlap DUPLEX_REGION (the tests' --region), moved onto a chr20 of DUPLEX_LEN
                            bases that starts at reference offset DUPLEX_SHIFT: one @SQ line, tid 0, pos / next_pos shifted.
                            Reads, motifs and the 100 kb interval keep their relative geometry. Indexed by tools/bamio.py.
duplex_window.fa(.fai)    = GRCh38_chr20.fa[DUPLEX_SHIFT : DUPLEX_SHIFT + DUPLEX_LEN] (line width and case kept)
duplex_hemi{,_nofilt}.bed = the reference goldens of `pileup-hemi` with the position columns (2, 3, 7, 8) shifted
"""
import os
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "tools"))
import bamio  # noqa: E402

OUT = os.path.join(HERE, "generated")

DUPLEX_REGION = (22613834, 22640468)    # chr20:22,613,835-22,640,468, 0-based half-open
DUPLEX_SHIFT = 22550000
DUPLEX_LEN = 140000


def duplex_window(res):
    b = bamio.Bam(res + "duplex_modcalls_sort.bam")
    chr20 = [n for n, _ in b.refs].index("chr20")
    lo, hi = DUPLEX_REGION

    def keep(r):
        f = bamio.rec_fields(r)
        beg, end = bamio.ref_span(f)
        return f["tid"] == chr20 and beg < hi and end > lo

    def shifted(r):
        f = bamio.rec_fields(r)
        beg, end = bamio.ref_span(f)
        assert DUPLEX_SHIFT <= beg and end <= DUPLEX_SHIFT + DUPLEX_LEN
        next_tid, next_pos = struct.unpack_from("<ii", r, 20)
        if next_tid == chr20:
            next_tid, next_pos = 0, next_pos - DUPLEX_SHIFT
        elif next_tid >= 0:
            next_tid, next_pos = -1, -1
        pos = f["pos"] - DUPLEX_SHIFT
        return (struct.pack("<ii", 0, pos) + r[8:10] + struct.pack("<H", bamio.reg2bin(pos, end - DUPLEX_SHIFT)) + r[12:20]
                + struct.pack("<ii", next_tid, next_pos) + r[28:])

    b.records = [shifted(r) for r in b.records if keep(r)]
    lines = [ln for ln in b.header_text.decode().split("\n") if not ln.startswith("@SQ")]
    lines.insert(1, "@SQ\tSN:chr20\tLN:%d" % DUPLEX_LEN)
    b.header_text = "\n".join(lines).encode()
    b.refs = [("chr20", DUPLEX_LEN)]
    b.write(os.path.join(OUT, "duplex_window.bam"), level=9, index=True)

    # FASTA slice: same line width, same case
    with open(res + "GRCh38_chr20.fa") as fa:
        fa.readline()
        width = len(fa.readline().rstrip("\n"))
        fa.seek(0)
        fa.readline()
        seq = fa.read().replace("\n", "")[DUPLEX_SHIFT:DUPLEX_SHIFT + DUPLEX_LEN]
    hdr = ">chr20\n"
    with open(os.path.join(OUT, "duplex_window.fa"), "w") as out:
        out.write(hdr)
        for i in range(0, len(seq), width):
            out.write(seq[i:i + width] + "\n")
    with open(os.path.join(OUT, "duplex_window.fa.fai"), "w") as out:
        out.write("chr20\t%d\t%d\t%d\t%d\n" % (DUPLEX_LEN, len(hdr), width, width + 1))
    for name in ("duplex_hemi.bed", "duplex_hemi_nofilt.bed"):
        with open(res + name) as src, open(os.path.join(OUT, name), "w") as dst:
            for ln in src:
                c = ln.split("\t")
                for k in (1, 2, 6, 7):
                    c[k] = str(int(c[k]) - DUPLEX_SHIFT)
                dst.write("\t".join(c))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    os.makedirs(OUT, exist_ok=True)
    duplex_window(os.path.join(sys.argv[1], "tests", "resources") + os.sep)
    for f in ("duplex_window.bam", "duplex_window.bam.bai", "duplex_window.fa", "duplex_window.fa.fai", "duplex_hemi.bed", "duplex_hemi_nofilt.bed"):
        os.chmod(os.path.join(OUT, f), 0o644)
