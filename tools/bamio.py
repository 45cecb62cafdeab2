"""Tiny pure-Python BGZF/BAM reader + writer for tests and fixture preparation (no pysam/htslib here).

Only what the tests need: iterate records, look at / rewrite aux tags, build records of an exact shape (make_record,
mm_for), write a coordinate-sorted BAM back out (BGZF members of <= 64 KiB, EOF marker) and a FASTA with its .fai.
Not used by the product path.
"""
import struct
import zlib

BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def read_bgzf(path):
    data = open(path, "rb").read()
    out = []
    off = 0
    while off < len(data):
        xlen = struct.unpack_from("<H", data, off + 10)[0]
        x = off + 12
        bsize = None
        while x < off + 12 + xlen:
            si1, si2, slen = data[x], data[x + 1], struct.unpack_from("<H", data, x + 2)[0]
            if si1 == 66 and si2 == 67:
                bsize = struct.unpack_from("<H", data, x + 4)[0]
            x += 4 + slen
        clen = bsize + 1
        out.append(zlib.decompress(data[off + 12 + xlen: off + clen - 8], -15))
        off += clen
    return b"".join(out)


class Bam:
    def __init__(self, path=None):
        self.header_text = b""
        self.refs = []      # (name, length)
        self.records = []   # raw record bytes (without block_size)
        if path:
            self.load(path)

    def load(self, path):
        raw = read_bgzf(path)
        assert raw[:4] == b"BAM\x01"
        l_text = struct.unpack_from("<I", raw, 4)[0]
        self.header_text = raw[8:8 + l_text]
        o = 8 + l_text
        n_ref = struct.unpack_from("<I", raw, o)[0]
        o += 4
        for _ in range(n_ref):
            ln = struct.unpack_from("<I", raw, o)[0]
            name = raw[o + 4:o + 4 + ln - 1].decode()
            length = struct.unpack_from("<I", raw, o + 4 + ln)[0]
            self.refs.append((name, length))
            o += 8 + ln
        while o + 4 <= len(raw):
            bs = struct.unpack_from("<I", raw, o)[0]
            self.records.append(raw[o + 4:o + 4 + bs])
            o += 4 + bs

    def write(self, path, level=6, index=False):
        """index=True also writes path + ".bai" (the records must be coordinate sorted)."""
        parts = [b"BAM\x01", struct.pack("<I", len(self.header_text)), self.header_text, struct.pack("<I", len(self.refs))]
        for name, length in self.refs:
            nb = name.encode() + b"\x00"
            parts += [struct.pack("<I", len(nb)), nb, struct.pack("<I", length)]
        rec_off = []            # offset of every record's block_size in the inflated stream
        o = sum(len(x) for x in parts)
        for r in self.records:
            rec_off.append(o)
            o += 4 + len(r)
            parts += [struct.pack("<I", len(r)), r]
        raw = b"".join(parts)
        member_off = []         # compressed offset of every member; member k holds raw[k * 0xff00 : (k + 1) * 0xff00]
        with open(path, "wb") as f:
            for i in range(0, len(raw), 0xff00):
                member_off.append(f.tell())
                chunk = raw[i:i + 0xff00]
                co = zlib.compressobj(level, zlib.DEFLATED, -15)
                comp = co.compress(chunk) + co.flush()
                bsize = len(comp) + 25
                f.write(struct.pack("<BBBBIBBHBBHH", 31, 139, 8, 4, 0, 0, 255, 6, 66, 67, 2, bsize))
                f.write(comp)
                f.write(struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))
            member_off.append(f.tell())
            f.write(BGZF_EOF)
        if index:
            def voff(u):
                k = u // 0xff00
                return member_off[k] << 16 | (u % 0xff00) if k < len(member_off) - 1 else member_off[-1] << 16
            ends = rec_off[1:] + [len(raw)]
            write_bai(path + ".bai", len(self.refs), [(rec_fields(r), voff(b), voff(e)) for r, b, e in zip(self.records, rec_off, ends)])


def ref_span(f):
    """[beg, end) on the reference of a record's fields (rec_fields); unmapped or zero-length: one base, as htslib indexes it."""
    rl = sum(c >> 4 for c in f["cigar"] if (c & 15) in (0, 2, 3, 7, 8))
    return f["pos"], f["pos"] + (rl if rl and not f["flag"] & 4 else 1)


def reg2bin(beg, end):
    end -= 1
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return base + (beg >> shift)
    return 0


def write_bai(path, n_ref, recs):
    """BAI (SAMv1 5.2) of coordinate-sorted records [(fields, voffset begin, voffset end)]: bins with their chunks (contiguous
    chunks merged), the 37450 pseudo-bin (offset range, mapped / unmapped counts), the 16 kb linear index (windows without a
    record take the previous window's offset), and the count of records without coordinates."""
    refs = [dict(bins={}, lin=[], beg=None, end=0, n_map=0, n_unmap=0) for _ in range(n_ref)]
    n_no_coor = 0
    for f, vb, ve in recs:
        if f["tid"] < 0:
            n_no_coor += 1
            continue
        R = refs[f["tid"]]
        beg, end = ref_span(f)
        ch = R["bins"].setdefault(reg2bin(beg, end), [])
        if ch and ch[-1][1] == vb:
            ch[-1][1] = ve
        else:
            ch.append([vb, ve])
        for w in range(beg >> 14, ((end - 1) >> 14) + 1):
            if len(R["lin"]) <= w:
                R["lin"] += [None] * (w + 1 - len(R["lin"]))
            if R["lin"][w] is None:
                R["lin"][w] = vb
        R["beg"] = vb if R["beg"] is None else R["beg"]
        R["end"] = ve
        R["n_unmap" if f["flag"] & 4 else "n_map"] += 1
    out = [b"BAI\x01", struct.pack("<I", n_ref)]
    for R in refs:
        any_rec = R["n_map"] + R["n_unmap"] > 0
        out.append(struct.pack("<I", len(R["bins"]) + (1 if any_rec else 0)))
        for b in sorted(R["bins"]):
            out.append(struct.pack("<II", b, len(R["bins"][b])) + b"".join(struct.pack("<QQ", x, y) for x, y in R["bins"][b]))
        if any_rec:
            out.append(struct.pack("<IIQQQQ", 37450, 2, R["beg"], R["end"], R["n_map"], R["n_unmap"]))
        lin = R["lin"]
        for w in range(len(lin)):
            if lin[w] is None:
                lin[w] = lin[w - 1] if w else 0
        out.append(struct.pack("<I", len(lin)) + b"".join(struct.pack("<Q", v) for v in lin))
    out.append(struct.pack("<Q", n_no_coor))
    with open(path, "wb") as fh:
        fh.write(b"".join(out))


def rec_fields(r):
    tid, pos, l_name, mapq, bin_, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", r, 0)
    o = 32
    name = r[o:o + l_name - 1].decode()
    o += l_name
    cigar = list(struct.unpack_from("<%dI" % n_cig, r, o))
    o += 4 * n_cig
    seq = r[o:o + (l_seq + 1) // 2]
    o += (l_seq + 1) // 2
    qual = r[o:o + l_seq]
    o += l_seq
    return dict(tid=tid, pos=pos, flag=flag, l_seq=l_seq, name=name, cigar=cigar, seq=seq, qual=qual, aux_off=o)


def iter_aux(r, o):
    """yields (tag, type, start, end) with start/end spanning the whole field"""
    n = len(r)
    while o + 3 <= n:
        tag = r[o:o + 2]
        ty = chr(r[o + 2])
        p = o + 3
        if ty in "AcC":
            e = p + 1
        elif ty in "sS":
            e = p + 2
        elif ty in "iIf":
            e = p + 4
        elif ty in "ZH":
            e = r.index(b"\x00", p) + 1
        elif ty == "B":
            sub = chr(r[p])
            cnt = struct.unpack_from("<I", r, p + 1)[0]
            es = 1 if sub in "cC" else 2 if sub in "sS" else 4
            e = p + 5 + es * cnt
        else:
            raise ValueError("bad aux type " + ty)
        yield tag, ty, o, e
        o = e


def get_aux(r, tag):
    f = rec_fields(r)
    for t, ty, s, e in iter_aux(r, f["aux_off"]):
        if t == tag:
            if ty == "Z":
                return r[s + 3:e - 1]
            if ty == "B":
                return r[s + 8:e]
            return r[s + 3:e]
    return None


def replace_aux(r, mapping):
    """mapping: old tag (bytes) -> (new tag, type char, payload bytes) or None to drop"""
    f = rec_fields(r)
    out = [r[:f["aux_off"]]]
    for t, ty, s, e in iter_aux(r, f["aux_off"]):
        if t in mapping:
            new = mapping[t]
            if new is None:
                continue
            if callable(new):
                new = new(ty, r[s + 3:e])
            ntag, nty, payload = new
            out.append(ntag + nty.encode() + payload)
        else:
            out.append(r[s:e])
    return b"".join(out)


CIGAR_OPS = "MIDNSHP=X"
SEQ_NIB = "=ACMGRSVTWYHKDBN"
COMPLEMENT = str.maketrans("ACGTRYKMSWBVDHN", "TGCAYRMKSWVBHDN")


def revcomp(seq):
    return seq.translate(COMPLEMENT)[::-1]


def cigar_spans(cigar):
    """(query length, reference length) consumed by a [(op char, len)] CIGAR."""
    return (sum(n for op, n in cigar if op in "MIS=X"), sum(n for op, n in cigar if op in "MDN=X"))


def aux_z(tag, text):
    return tag.encode() + b"Z" + (text.encode() if isinstance(text, str) else text) + b"\x00"


def aux_b(tag, sub, values):
    fmt = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[sub]
    return tag.encode() + b"B" + sub.encode() + struct.pack("<I%d%s" % (len(values), fmt), len(values), *values)


def aux_i(tag, value):
    return tag.encode() + b"i" + struct.pack("<i", value)


def make_record(tid, pos, flag, cigar, seq, mm=None, ml=None, aux=(), name="r", long_cigar=False, cg_at="last", mapq=60):
    """Raw bytes (without block_size) of one BAM record.

    cigar: [(op char, len)]; seq: bases, IUPAC letters allowed, "" for SEQ *; qualities are 0xff. mm / ml: the MM text and
    the ML probabilities (ints 0-255) in read orientation, or None to leave the tags out; aux: further encoded fields
    (aux_z, aux_i, aux_b), written after MM/ML. long_cigar=True stores the CIGAR in CG:B,I with the SAMv1 4.2.2 placeholder
    `<l_seq>S <ref_len>N` in the core; cg_at puts the CG field "first", "middle" (between MM and ML) or "last"."""
    ops = [(CIGAR_OPS.index(op), n) for op, n in cigar]
    words = [n << 4 | op for op, n in ops]
    _, rlen = cigar_spans(cigar)
    core = [len(seq) << 4 | 4, rlen << 4 | 3] if long_cigar else words
    end = pos + (rlen if rlen and not flag & 4 else 1)
    nb = name.encode() + b"\x00"
    packed = bytearray((len(seq) + 1) // 2)
    for i, c in enumerate(seq):
        packed[i >> 1] |= SEQ_NIB.index(c.upper()) << (0 if i & 1 else 4)
    fields = []
    if mm is not None:
        fields.append(aux_z("MM", mm))
    if ml is not None:
        fields.append(aux_b("ML", "C", list(ml)))
    if long_cigar:
        cg = aux_b("CG", "I", words)
        fields.insert({"first": 0, "middle": 1 if mm is not None else 0, "last": len(fields)}[cg_at], cg)
    fields += list(aux)
    head = struct.pack("<iiBBHHHiiii", tid, pos, len(nb), mapq, reg2bin(pos, end), len(core), flag, len(seq), -1, -1, 0)
    return head + nb + struct.pack("<%dI" % len(core), *core) + bytes(packed) + b"\xff" * len(seq) + b"".join(fields)


def mm_for(seq, rev, lists):
    """MM text and ML values for calls given in read orientation.

    seq: the stored (reference-orientation) SEQ; rev: the record is reverse (the read is the reverse complement of seq).
    lists: [(header, calls)] with header such as "C+m?" or "C+hm." and calls [(read position, prob or (prob per code))],
    every position a base of the list's fundamental base in read orientation (any base for N). The deltas count exact
    base letters only, as the MM spec does; probabilities of a multi-code list are interleaved per call."""
    read = revcomp(seq) if rev else seq
    texts, ml = [], []
    for header, calls in lists:
        base = header[0]
        occ = [i for i, c in enumerate(read) if base == "N" or c.upper() == base]
        rank = {q: k for k, q in enumerate(occ)}
        last, deltas = -1, []
        for q, p in sorted(calls, key=lambda c: c[0]):
            k = rank[q]
            deltas.append(k - last - 1)
            last = k
            ml += list(p) if isinstance(p, (tuple, list)) else [p]
        texts.append(header + "".join("," + str(d) for d in deltas) + ";")
    return "".join(texts), ml


def write_fasta(path, contigs, width=60):
    """FASTA of {name: sequence} plus its samtools-style .fai (name, length, offset, bases and bytes per line)."""
    with open(path, "w") as fa, open(path + ".fai", "w") as fai:
        off = 0
        for name, s in contigs.items():
            head = ">%s\n" % name
            off += len(head)
            fai.write("%s\t%d\t%d\t%d\t%d\n" % (name, len(s), off, width, width + 1))
            body = "".join(s[i:i + width] + "\n" for i in range(0, len(s), width))
            fa.write(head + body)
            off += len(body)


def bam_of(refs, records, header_text=b""):
    """A Bam of [(name, length)] refs and raw records, sorted by (tid, pos) the way a coordinate-sorted BAM is
    (unplaced records last); write it with .write(path, index=True)."""
    b = Bam()
    b.refs = list(refs)
    b.header_text = header_text or ("@HD\tVN:1.6\tSO:coordinate\n" + "".join("@SQ\tSN:%s\tLN:%d\n" % r for r in refs)).encode()
    key = lambda r: (struct.unpack_from("<i", r, 0)[0] % (1 << 31), struct.unpack_from("<i", r, 4)[0])
    b.records = sorted(records, key=key)
    return b
