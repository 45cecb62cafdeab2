"""An independent column-wise model of `modkit pileup` (reference v0.4.4): reads -> columns -> features -> tallies -> rows ->
bedMethyl text, in plain Python, written from the reference's Rust sources and following their loop structure (one position
at a time, one alignment at a time):

    columns, admission, qpos          process_region / PileupIter (pileup/mod.rs:577-604, 718-1020); htslib's default
                                      pileup mask 0x4|0x100|0x200|0x400, then record_is_not_primary (util.rs:405-407)
                                      and seq_len == 0 (pileup/mod.rs:783-791)
    read cache                        ReadCache::add_record / get_mod_call / add_mod_codes_for_record (read_cache.rs:111-355)
    forward aligned pairs             get_aligned_pairs_forward (util.rs:122-145)
    edge filter                       edge_filter_positions, EdgeFilter (mod_bam.rs:1075-1102, 1641-1671)
    features, strand rules            Feature, FeatureVector::add_feature (pileup/mod.rs:29-52, 238-281), get_forward_read_base (:612-624)
    tallies, rows                     Tally, diff_calls_count, add_tally_to_counts, decode (:167-224, 283-445)
    --combine-strands                 combine_strand_features, combine_counts_ignore_strand (:469-561, 93-137)
    focus positions                   find_motif_hits, MotifInfo (find_motifs/motif_bed.rs:21-337); the per-interval sequence
                                      search and its --combine-strands extension (fasta.rs:42-226); FocusPositions
                                      (interval_chunks.rs:32-408); the interval feeder (interval_chunks.rs:563-643)
    --include-bed                     StrandedPositionFilter (position_filter.rs:20-45, 230-300)
    --partition-tag                   parse_tags_from_record (pileup/mod.rs:626-643, 795-830)
    text                              BedMethylWriter::write_feature_counts (writers.rs:87-156)

MM / ML decoding is mmmodel.mod_base_info and the per-call arithmetic is callmodel; both are independent models of their own.

Where this project knowingly differs from the reference, or where the model does not follow it, the corpus keeps clear of the
case (DESIGN.md section 7 states the same):

    case                                                  reference                             here / the model
    --max-depth (htslib's per-interval read buffer)       drops reads past the depth            not modelled: columns stay
                                                                                                below 8 000 reads
    two records with one read name in one interval        the read cache keys on the name:      not replicated (SURVEY B.3);
                                                          the second record reuses the first's  the corpus names every
                                                          calls                                 record uniquely
    a CpG whose C and G lie in different intervals        not a motif position (the motif       the same: the model searches
    (without --combine-strands)                           search runs on each interval's        each interval's sequence
                                                          sequence)
    two primary bases calling one code at one column      rows of equal (strand, code) in       the corpus keeps every code on
                                                          hash order                            one primary base
"""
import bisect
import re

import numpy as np

import bamio
import callmodel as cm
import mmmodel as mm

F32 = np.float32
COMP = {"A": "T", "C": "G", "G": "C", "T": "A"}
NIB = "=ACMGRSVTWYHKDBN"
HTS_MASK = 0x4 | 0x100 | 0x200 | 0x400       # htslib pileup's default read filter
NOT_PRIMARY = 0x100 | 0x800 | 0x400          # record_is_not_primary: supplementary, secondary, duplicate
POS, NEG = "+", "-"
BOTH = "."                                   # StrandRule::Both (its char form)


def code_key(code):
    """ModCodeRepr's derived Ord: every letter code before every ChEBI code."""
    return (1, code) if isinstance(code, int) else (0, code)


# ---------------------------------------------------------------------------------------------------------------------------
# options

class Options:
    """The pileup flags the model reads (a subset of the CLI, spelled as the CLI spells them)."""

    def __init__(self, args):
        a = list(args)
        if "--preset" in a and a[a.index("--preset") + 1] == "traditional":   # the preset's flags (pileup/subcommand.rs)
            a += ["--cpg", "--ignore", "h", "--combine-strands"]
        val = lambda k: [a[i + 1] for i, x in enumerate(a) if x == k]
        self.interval = int((val("-i") or val("--interval-size") or ["100000"])[-1])
        self.force = "--force-allow-implicit" in a
        self.combine_mods = "--combine-mods" in a
        self.combine_strands = "--combine-strands" in a
        self.ignore = (val("--ignore") or [None])[-1]
        self.mixed_delim = "--mixed-delim" in a or "--mixed-delimiters" in a
        self.header = "--with-header" in a or "--header" in a
        self.region = (val("--region") or [None])[-1]
        self.partition_tags = val("--partition-tag")
        self.ref = (val("--ref") or [None])[-1]
        self.include_bed = (val("--include-bed") or val("--include-positions") or [None])[-1]
        motifs = [(a[i + 1], int(a[i + 2])) for i, x in enumerate(a) if x == "--motif"]
        if "--cpg" in a and ("CG", 0) not in motifs:                 # RegexMotif::from_raw_parts (motif_bed.rs:167-179)
            motifs.append(("CG", 0))
        self.motifs = motifs
        edge = (val("--edge-filter") or [None])[-1]
        self.edge = None
        if edge is not None:
            s, _, e = edge.partition(",")
            self.edge = (int(s), int(e or s), "--invert-edge-filter" in a)
        per_mod = dict(v.split(":") for v in val("--mod-thresholds"))
        per_base, default = {}, 0.0
        for v in val("--filter-threshold"):
            if ":" in v:
                b, t = v.split(":")
                per_base[b] = float(t)
            else:
                default = float(v)
        if "--no-filtering" not in a and not val("--filter-threshold") and not per_mod:
            raise ValueError("the model takes thresholds as inputs: pass --no-filtering, --filter-threshold or --mod-thresholds")
        self.caller = cm.Caller(per_mod, per_base, default)


# ---------------------------------------------------------------------------------------------------------------------------
# reads

class Read:
    """One BAM record: core fields, the stored SEQ as letters, the CIGAR as (op, length), the MM / ML tags and the raw record."""

    def __init__(self, raw):
        f = bamio.rec_fields(raw)
        self.raw, self.tid, self.pos, self.flag, self.name = raw, f["tid"], f["pos"], f["flag"], f["name"]
        self.cigar = [("MIDNSHP=X"[c & 15], c >> 4) for c in f["cigar"]]
        s = f["seq"]
        self.seq = "".join(NIB[(s[i >> 1] >> (0 if i & 1 else 4)) & 15] for i in range(f["l_seq"]))
        self.rev = bool(self.flag & 0x10)
        self.mm = bamio.get_aux(raw, b"MM")
        self.mm = bamio.get_aux(raw, b"Mm") if self.mm is None else self.mm
        ml = bamio.get_aux(raw, b"ML")
        ml = bamio.get_aux(raw, b"Ml") if ml is None else ml
        self.ml = list(ml) if ml is not None else []
        self.end = self.pos + sum(n for op, n in self.cigar if op in "MDN=X")

    def columns(self, start, end):
        """[(reference position, what htslib's pileup reports for this alignment there)] over [start, end): ("base", qpos),
        ("del", None) or ("skip", None) (is_refskip)."""
        out, r, q = [], self.pos, 0
        for op, n in self.cigar:
            if op in "M=X":
                out += [(p, ("base", q + p - r)) for p in range(max(r, start), min(r + n, end))]
                r, q = r + n, q + n
            elif op == "D" or op == "N":
                out += [(p, ("del" if op == "D" else "skip", None)) for p in range(max(r, start), min(r + n, end))]
                r += n
            elif op in "IS":
                q += n
        return out

    def aligned_pairs_forward(self):
        """{forward query position: reference position} of the M / = / X bases (util.rs:122-145)."""
        out, r, q, n_seq = {}, self.pos, 0, len(self.seq)
        for op, n in self.cigar:
            if op in "M=X":
                for k in range(n):
                    out[(n_seq - 1 - (q + k)) if self.rev else q + k] = r + k
                r, q = r + n, q + n
            elif op in "DN":
                r += n
            elif op in "IS":
                q += n
        return out

    def partition_key(self, tags):
        """parse_tags_from_record (pileup/mod.rs:626-643): the values joined by `_`, "missing" for an absent tag, None when
        no tag is present. Only Z / A / integer tags are read."""
        vals = []
        f = bamio.rec_fields(self.raw)
        found = {t: (ty, self.raw[s + 3:e]) for t, ty, s, e in bamio.iter_aux(self.raw, f["aux_off"])}
        for tag in tags:
            x = found.get(tag.encode())
            if x is None:
                vals.append(None)
            elif x[0] == "Z":
                vals.append(x[1][:-1].decode())
            elif x[0] == "A":
                vals.append(chr(x[1][0]))
            else:
                vals.append(str(int.from_bytes(x[1], "little", signed=x[0] in "csi")))
        if all(v is None for v in vals):
            return None
        return "_".join("missing" if v is None else v for v in vals)


class ReadState:
    """The read cache's entries for one read: `calls[strand][dna_base] = {reference position: call}` (strand of the MM list)
    and `codes[reference strand][threshold base] = set of codes`; `skipped` when the read is in the skip set."""

    def __init__(self):
        self.calls, self.codes, self.skipped = {POS: {}, NEG: {}}, {POS: {}, NEG: {}}, False


def add_record(read, opts):
    """ReadCache::add_record (read_cache.rs:111-211)."""
    st = ReadState()
    fwd = bamio.revcomp(read.seq) if read.rev else read.seq
    try:
        tables = mm.mod_base_info(read.mm, read.ml, fwd) if read.mm is not None else {}
    except cm.ReadError:
        tables = None
    if not tables or (any(t.mode == mm.DEFAULT for t in tables.values()) and not opts.force):   # :115-137
        st.skipped = True
        return st
    ar, pairs, added = cm.Arith(False), None, False
    for (strand, dna_base), t in tables.items():
        try:
            maps = cm.position_maps([([cm.code_of(str(c)) for c in codes], v) for codes, v in t.lists], ar) if t.lists else {}
        except cm.ReadError:                                            # ProbaGreaterThanOne: the whole read fails
            st.skipped = True
            return st
        for p, codes in t.inferred.items():                             # inferred canonical entries (mod_bam.rs:1265-1292)
            m = cm.FxMap(reserve=len(codes))
            for code in codes:
                m.insert(cm.code_of(str(code)), ar.num(0.0))
            maps[p] = m
        threshold_base = dna_base if strand == POS else COMP[dna_base]   # :147-150
        if opts.edge is not None:                                        # :151-165
            s, e, inverted = opts.edge
            n = len(read.seq)
            if n <= s or n <= e:
                continue
            keep = (lambda p: p < s or p >= n - e) if inverted else (lambda p: s <= p < n - e)
            maps = {p: m for p, m in maps.items() if keep(p)}
            if not maps:
                continue
        if opts.ignore is not None:                                      # into_collapsed (:167-169)
            maps = {p: cm.redistribute(m, cm.code_of(opts.ignore), ar) for p, m in maps.items()}
        codes = set()
        for m in maps.values():                                          # :171-179
            codes |= {c for c, _ in m.items()}
        ref_strand = POS if (strand == POS) != read.rev else NEG         # :181-188
        st.codes[ref_strand].setdefault(threshold_base, set()).update(codes)
        pairs = read.aligned_pairs_forward() if pairs is None else pairs
        st.calls[strand][dna_base] = {pairs[q]: cm.call(m, opts.caller, threshold_base, ar) for q, m in maps.items() if q in pairs}
        added = True
    st.skipped = not added                                               # :206-210
    return st


# ---------------------------------------------------------------------------------------------------------------------------
# features and tallies

DELETE, FILTERED = ("delete",), ("filtered",)


def nocall(base):
    return ("nocall", base)


def feature_of(call, read_base):
    """Feature::from_base_mod_call (pileup/mod.rs:38-51); `call` as callmodel.call returns it."""
    if call[0] == "fail":
        return FILTERED
    if call[0] == "canonical":
        return ("modcall", ("canonical", read_base), read_base)
    return ("modcall", ("mod", call[1]), read_base)


class Tally:
    def __init__(self):
        self.n_delete, self.n_filtered, self.basecall_counts, self.modcall_counts = 0, 0, {}, {}

    def add_feature(self, f):                                            # :177-193
        if f == FILTERED:
            self.n_filtered += 1
        elif f == DELETE:
            self.n_delete += 1
        elif f[0] == "modcall":
            states = self.modcall_counts.setdefault(f[2], {})
            states[f[1]] = states.get(f[1], 0) + 1
        else:
            self.basecall_counts[f[1]] = self.basecall_counts.get(f[1], 0) + 1

    def diff_calls_count(self, primary):                                 # :198-223
        return (sum(n for b, n in self.basecall_counts.items() if b != primary)
                + sum(sum(s.values()) for b, s in self.modcall_counts.items() if b != primary))


class Row:
    __slots__ = ("strand", "code", "cov", "n_mod", "n_canon", "n_other", "n_delete", "n_fail", "n_diff", "n_nocall", "motif", "primary")

    def __init__(self, strand, code, cov, n_mod, n_canon, n_other, n_delete, n_fail, n_diff, n_nocall, motif):
        (self.strand, self.code, self.cov, self.n_mod, self.n_canon, self.n_other, self.n_delete, self.n_fail, self.n_diff,
         self.n_nocall, self.motif) = strand, code, cov, n_mod, n_canon, n_other, n_delete, n_fail, n_diff, n_nocall, motif
        self.primary = None

    def counts(self):
        return (self.cov, self.n_mod, self.n_canon, self.n_other, self.n_delete, self.n_fail, self.n_diff, self.n_nocall)

    def __repr__(self):
        return "Row(%s, %r, %r, motif=%r)" % (self.strand, self.code, self.counts(), self.motif)


class FeatureVector:
    """FeatureVector (pileup/mod.rs:226-446). `delete_strand` is the read strand a deletion is added with (Positive in the
    reference); tests set it to put a known mistake into the model."""
    delete_strand = POS

    def __init__(self):
        self.pos_tally, self.neg_tally = Tally(), Tally()

    def add_feature(self, alignment_strand, feature, read_strand, rule):  # :238-281
        same = alignment_strand == read_strand
        if rule == BOTH:
            (self.pos_tally if same else self.neg_tally).add_feature(feature)
        elif rule == POS:
            if same:
                self.pos_tally.add_feature(feature)
        elif not same:
            self.neg_tally.add_feature(feature)

    @staticmethod
    def add_tally_to_counts(out, tally, strand, observed, combine_mods, motif_idxs):   # :283-410
        for primary, states in tally.modcall_counts.items():
            n_nocall = tally.basecall_counts.get(primary, 0)
            n_canonical = sum(n for s, n in states.items() if s[0] == "canonical")
            mod_calls = {}
            for s, n in states.items():
                if s[0] == "mod":
                    mod_calls[s[1]] = mod_calls.get(s[1], 0) + n
            total_mod = sum(mod_calls.values())
            cov = total_mod + n_canonical
            n_diff = tally.diff_calls_count(primary)
            idxs = motif_idxs if motif_idxs is not None else [None]
            first = len(out)
            if combine_mods:
                for idx in idxs:
                    out.append(Row(strand, primary, cov, total_mod, n_canonical, 0, tally.n_delete, tally.n_filtered, n_diff, n_nocall, idx))
            else:
                for code in observed.get(primary, set()):
                    n_mod = mod_calls.get(code, 0)
                    for idx in idxs:
                        out.append(Row(strand, code, cov, n_mod, n_canonical, max(total_mod - n_mod, 0), tally.n_delete,
                                       tally.n_filtered, n_diff, n_nocall, idx))
            for r in out[first:]:
                r.primary = primary

    def decode(self, pos_observed, neg_observed, combine_mods, pos_motifs, neg_motifs):   # :412-445
        out = []
        self.add_tally_to_counts(out, self.pos_tally, POS, pos_observed, combine_mods, pos_motifs)
        self.add_tally_to_counts(out, self.neg_tally, NEG, neg_observed, combine_mods, neg_motifs)
        out.sort(key=lambda r: (r.strand, code_key(r.code)))            # stable, as slice::sort_by
        return out


# ---------------------------------------------------------------------------------------------------------------------------
# focus positions

IUPAC = {"A": "A", "C": "C", "G": "G", "T": "T", "U": "U", "M": "[AC]", "R": "[AG]", "W": "[AT]", "S": "[CG]", "Y": "[CT]",
         "K": "[GT]", "V": "[ACG]", "H": "[ACT]", "D": "[AGT]", "B": "[CGT]", "X": "[ACGT]", "N": "[ACGT]"}


class Motif:
    """RegexMotif::parse_string (motif_bed.rs:197-223) and MotifInfo (:111-141)."""

    def __init__(self, raw, offset):
        self.raw, self.fwd_off, self.length = raw, offset, len(raw)
        self.fwd = "".join(IUPAC[c] for c in raw)
        self.rc = "".join({"A": "T", "C": "G", "G": "C", "T": "A", "U": "A", "[": "]", "]": "["}.get(c, c) for c in self.fwd[::-1])
        self.rev_off = len(raw) - (offset + 1)
        self.palindrome = self.fwd == self.rc
        self.label = "%s,%d" % (raw, offset)

    def negative_strand_position(self, p):                               # :124-140
        if not self.palindrome:
            return None
        adj = p + self.rev_off - self.fwd_off
        return adj if adj >= 0 else None

    def hits(self, seq):
        """find_motif_hits (:288-337): [(position, strand)], overlapping matches of fixed-length patterns."""
        starts = lambda pat: [m.start() for m in re.finditer("(?=%s)" % pat, seq)]
        out = []
        if self.palindrome:
            for s in starts(self.fwd):
                pair = [(s + self.fwd_off, POS), (s + self.rev_off, NEG)]
                out += pair if self.fwd_off <= self.rev_off else pair[::-1]
        elif self.length == 1:
            fw, rv = self.fwd, COMP[self.fwd]
            out = [(i, POS if c == fw else NEG) for i, c in enumerate(seq) if c in (fw, rv)]
        else:
            out = [(s + self.fwd_off, POS) for s in starts(self.fwd)] + [(s + self.rev_off, NEG) for s in starts(self.rc)]
            out.sort(key=lambda x: x[0])
        return out


def absorb(rule, strand):                                                # StrandRule::absorb (util.rs:336-344)
    return rule if rule == strand else BOTH


def combine(rule, other):                                                # StrandRule::combine (util.rs:346-352)
    return rule if rule == other else BOTH


class IncludeBed:
    """StrandedPositionFilter::from_bed_file (position_filter.rs:230-300): BED3 lines cover both strands, BED6 lines the
    strand of column 6 (`.` both)."""

    def __init__(self, path, names):
        self.iv = {POS: {}, NEG: {}}
        for line in open(path):
            parts = line.split()
            if len(parts) < 3 or parts[0] not in names or not parts[1].isdigit() or not parts[2].isdigit():
                continue
            if len(parts) == 3:
                strands = (POS, NEG)
            elif len(parts) >= 6 and parts[5] in "+-.":
                strands = {"+": (POS,), "-": (NEG,), ".": (POS, NEG)}[parts[5]]
            else:
                continue
            for s in strands:
                self.iv[s].setdefault(names[parts[0]], []).append((int(parts[1]), int(parts[2])))

    def contains(self, tid, pos, strand):                                # :27-43
        return any(a <= pos < b for a, b in self.iv[strand].get(tid, ()))


def motif_locations(motifs, seq, start, tid, include):
    """get_motifs_on_seq (fasta.rs:42-90): per motif {position: rule} of the hits on `seq` (placed at `start`), filtered
    strand-wise by the include-bed."""
    out = []
    for m in motifs:
        locs = {}
        for p, strand in m.hits(seq):
            p += start
            if include is not None and not include.contains(tid, p, strand):
                continue
            locs[p] = absorb(locs[p], strand) if p in locs else strand
        out.append(locs)
    return out


class Focus:
    """FocusPositions of one interval: `rules` {position: rule} (None: all positions), `pos_ids` / `neg_ids` {position:
    [motif index]}, `pos_motifs` {position: [motif index]} of MotifCombineStrands."""

    def __init__(self):
        self.rules, self.pos_ids, self.neg_ids, self.pos_motifs = None, {}, {}, None

    def check(self, p):                                                  # check_position (interval_chunks.rs:352-374)
        return BOTH if self.rules is None else self.rules.get(p)


def focus_motif(motifs, locs, start, end):
    """FocusPositions::new_motif (interval_chunks.rs:62-202)."""
    f = Focus()
    f.rules = {}
    single = all(m.length == 1 for m in motifs)
    if len(motifs) == 1:
        for p, rule in sorted(locs[0].items()):
            if not start <= p < end:
                continue
            f.rules[p] = combine(f.rules[p], rule) if p in f.rules else rule
            if rule in (POS, BOTH):
                f.pos_ids[p] = [0]
            if rule in (NEG, BOTH):
                f.neg_ids[p] = [0]
    elif single:                                                         # add_single_base_motifs (:204-248)
        ids = {m.raw: k for k, m in enumerate(motifs)}
        for top, bottom in (("A", "T"), ("C", "G")):
            if top not in ids:
                continue
            for p, rule in sorted(locs[ids[top]].items()):
                if not start <= p < end:
                    continue
                if bottom in ids:
                    f.rules[p] = BOTH
                    f.pos_ids[p] = f.neg_ids[p] = [ids[top], ids[bottom]]
                else:
                    f.rules[p] = rule
                    (f.pos_ids if rule == POS else f.neg_ids)[p] = [ids[top]]
    else:
        for k in range(len(motifs)):
            for p, rule in sorted(locs[k].items()):
                if not start <= p < end:
                    continue
                f.rules[p] = combine(f.rules[p], rule) if p in f.rules else rule
                if rule in (POS, BOTH):
                    f.pos_ids.setdefault(p, []).append(k)
                if rule in (NEG, BOTH):
                    f.neg_ids.setdefault(p, []).append(k)
    return f


def focus_motif_combine_strands(motifs, locs, start, end):
    """FocusPositions::new_motif_combine_strands (interval_chunks.rs:250-297)."""
    f = Focus()
    f.rules, f.pos_motifs = {}, {}
    for k in range(len(motifs)):
        for p, rule in sorted(locs[k].items()):
            if not start <= p < end:
                continue
            f.rules[p] = combine(f.rules[p], rule) if p in f.rules else rule
            if rule in (POS, BOTH):
                f.pos_motifs.setdefault(p, []).append(k)
            else:
                f.neg_ids.setdefault(p, []).append(k)
    f.pos_ids = f.pos_motifs
    return f


def focus_regions(include, tid, start, end):
    """FocusPositions::new_regions + check_position (interval_chunks.rs:299-374)."""
    f = Focus()
    f.rules = {}
    for p in range(start, end):
        hp, hn = include.contains(tid, p, POS), include.contains(tid, p, NEG)
        if hp or hn:
            f.rules[p] = BOTH if hp and hn else POS if hp else NEG
    return f


def intervals(opts, refs, fasta, include):
    """The interval feeder (interval_chunks.rs:563-643) with the motif search of each interval (fasta.rs:92-226):
    [(tid, start, end, Focus)]."""
    names = {n: k for k, (n, _) in enumerate(refs)}
    targets = [(k, 0, ln) for k, (_, ln) in enumerate(refs)]
    if opts.region is not None:
        name, _, span = opts.region.partition(":")
        tid = names[name]
        a, b = (int(x) for x in span.split("-")) if span else (0, refs[tid][1])
        targets = [(tid, a, min(b, refs[tid][1]))]
    motifs = [Motif(r, o) for r, o in opts.motifs]
    out = []
    for tid, cur, contig_end in targets:
        seq_all = fasta[refs[tid][0]].upper() if motifs else None
        while cur < contig_end:
            start, end = cur, min(cur + opts.interval, contig_end)
            if not motifs:
                f = Focus() if include is None else focus_regions(include, tid, start, end)
            elif not opts.combine_strands:
                f = focus_motif(motifs, motif_locations(motifs, seq_all[start:end], start, tid, include), start, end)
            else:
                longest = max(m.length for m in motifs)
                buf = longest * 5
                e_lim, e_buf = end, min(end + buf, contig_end)
                while True:                                              # fasta.rs:105-187
                    too_close = max(e_buf - longest, 0)
                    locs = motif_locations(motifs, seq_all[start:e_buf], start, tid, include)
                    ivs = sorted((p, p + (m.length - m.fwd_off)) for m, l in zip(motifs, locs) for p in l)
                    search_end = e_lim
                    merged = []
                    for a, b in ivs:
                        if merged and a <= merged[-1][1]:
                            merged[-1][1] = max(merged[-1][1], b)
                        else:
                            merged.append([a, b])
                    for a, b in merged:
                        if a < e_lim and b > e_lim - 1:
                            search_end = b
                            break
                    if search_end < too_close or e_buf >= contig_end:
                        locs = [{p: r for p, r in l.items() if p <= search_end} for l in locs]
                        end = min(search_end, contig_end)
                        break
                    e_lim, e_buf = e_buf, e_buf + buf
                f = focus_motif_combine_strands(motifs, locs, start, end)
            out.append((tid, start, end, f, motifs))
            cur = end
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# one run

def combine_strand_features(f, motifs, position_rows):
    """combine_strand_features (pileup/mod.rs:469-561): {position: {key: [Row]}} of the positive motif positions."""
    result = {}
    for p in sorted(f.pos_motifs):
        for idx in f.pos_motifs[p]:
            q = motifs[idx].negative_strand_position(p)
            if q is None:
                continue
            pm, nm = position_rows.get(p, {}), position_rows.get(q, {})
            for key in set(pm) | set(nm):
                feats = [r for r in pm.get(key, []) if r.strand == POS and r.motif == idx]
                feats += [r for r in nm.get(key, []) if r.strand == NEG and r.motif == idx]
                grouped = {}
                for r in feats:
                    grouped.setdefault(r.code, []).append(r)
                rows = result.setdefault(p, {}).setdefault(key, [])
                for code in sorted(grouped, key=code_key):
                    acc = Row(BOTH, code, 0, 0, 0, 0, 0, 0, 0, 0, idx)
                    for r in grouped[code]:                              # combine_counts_ignore_strand (:93-137)
                        acc = Row(BOTH, code, acc.cov + r.cov, acc.n_mod + r.n_mod, acc.n_canon + r.n_canon, acc.n_other + r.n_other,
                                  acc.n_delete + r.n_delete, acc.n_fail + r.n_fail, acc.n_diff + r.n_diff, acc.n_nocall + r.n_nocall, idx)
                    rows.append(acc)
    return result


def process_interval(reads, tid, start, end, f, motifs, opts, states):
    """process_region (pileup/mod.rs:718-1020): {position: {partition key: [Row]}}. `reads` are the records of the contig in
    file order; `states` the read cache (one add_record per read name, as the cache keys on the name)."""
    position_rows = {}
    columns = {}
    for r in reads:                                                      # htslib's columns of the interval, reads in file order
        if r.tid == tid and r.pos < end and r.end > start and not r.flag & HTS_MASK:
            for p, c in r.columns(start, end):
                columns.setdefault(p, []).append((r, c))
    for pos in range(start, end):
        rule = f.check(pos)
        if rule is None:
            continue
        column = [(r, c) for r, c in columns.get(pos, ())                 # the admission filter (:783-791)
                  if not (c[0] == "skip" or r.flag & NOT_PRIMARY or len(r.seq) == 0)]
        if not column:
            continue
        vectors, pos_codes, neg_codes = {}, {}, {}
        for r, (kind, qpos) in column:
            key = r.partition_key(opts.partition_tags) if opts.partition_tags else None
            fv = vectors.setdefault(key, FeatureVector())
            st = states.get(r.name)
            if st is None:
                st = states[r.name] = add_record(r, opts)
            if not st.skipped:                                           # add_mod_codes_for_record (read_cache.rs:299-355)
                for strand, dst in ((POS, pos_codes), (NEG, neg_codes)):
                    for base, codes in st.codes[strand].items():
                        dst.setdefault(key, {}).setdefault(base, set()).update(codes)
            else:
                pos_codes.setdefault(key, {}), neg_codes.setdefault(key, {})
            alignment_strand = NEG if r.rev else POS
            if kind == "del":
                fv.add_feature(alignment_strand, DELETE, FeatureVector.delete_strand, rule)
                continue
            b = r.seq[qpos]                                              # get_forward_read_base (:612-624)
            if b not in COMP:
                continue
            read_base = COMP[b] if r.rev else b
            pos_call = neg_call = None
            if not st.skipped:                                           # get_mod_call (read_cache.rs:232-297)
                pos_call = st.calls[POS].get(read_base, {}).get(pos)
                neg_call = st.calls[NEG].get(read_base, {}).get(pos)
            if pos_call is not None:
                fv.add_feature(alignment_strand, feature_of(pos_call, read_base), POS, rule)
            if neg_call is not None:
                fv.add_feature(alignment_strand, feature_of(neg_call, COMP[read_base]), NEG, rule)
            if pos_call is None and neg_call is None:
                fv.add_feature(alignment_strand, nocall(read_base), POS, rule)
        position_rows[pos] = {key: fv.decode(pos_codes.get(key, {}), neg_codes.get(key, {}), opts.combine_mods,
                                             f.pos_ids.get(pos), f.neg_ids.get(pos)) for key, fv in vectors.items()}
    if opts.combine_strands and f.pos_motifs is not None:
        position_rows = combine_strand_features(f, motifs, position_rows)
    return position_rows


def read_fasta(path):
    seqs, name = {}, None
    for line in open(path):
        line = line.rstrip("\n")
        if line.startswith(">"):
            name = line[1:].split()[0]
            seqs[name] = []
        elif name is not None:
            seqs[name].append(line)
    return {k: "".join(v) for k, v in seqs.items()}


def load_bam(path):
    b = bamio.Bam(path)
    return b.refs, [Read(raw) for raw in b.records]


def pileup(bam, args):
    """{partition key: [(contig name, position, Row)]} of a run, in output order (key None: no --partition-tag)."""
    opts = Options(args)
    refs, reads = load_bam(bam) if isinstance(bam, str) else bam
    fasta = read_fasta(opts.ref) if opts.ref else None
    include = IncludeBed(opts.include_bed, {n: k for k, (n, _) in enumerate(refs)}) if opts.include_bed else None
    by_tid = {}
    for r in reads:
        by_tid.setdefault(r.tid, []).append(r)
    starts = {t: [r.pos for r in rs] for t, rs in by_tid.items()}          # coordinate sorted
    span = {t: max(r.end - r.pos for r in rs) for t, rs in by_tid.items()}
    out = {}
    for tid, start, end, f, motifs in intervals(opts, refs, fasta, include):
        states = {}                                                      # one read cache per interval
        rs = by_tid.get(tid, [])
        if rs:                                                           # the records the interval's fetch returns
            rs = rs[bisect.bisect_left(starts[tid], start - span[tid]):bisect.bisect_left(starts[tid], end)]
        rows = process_interval(rs, tid, start, end, f, motifs, opts, states)
        for pos in sorted(rows):
            for key, rs in rows[pos].items():
                out.setdefault(key, []).extend((refs[tid][0], pos, r) for r in rs)
    return out, opts


def percent(row):
    """fraction_modified * 100 as f32, printed with {:.2}."""
    return "%.2f" % float(F32(F32(F32(row.n_mod) / F32(row.cov)) * F32(100.0)))


HEADER = "\t".join(["chrom", "chromStart", "chromEnd", "name", "score", "strand", "thickStart", "thickEnd", "color", "valid_coverage",
                    "percent_modified", "count_modified", "count_canonical", "count_other_mod", "count_delete", "count_fail",
                    "count_diff", "count_nocall"]) + "\n"


def text(rows, opts):
    """BedMethylWriter (writers.rs:74-156) of one key's rows."""
    labels = [Motif(r, o).label for r, o in opts.motifs]
    space = " " if opts.mixed_delim else "\t"
    out = [HEADER] if opts.header else []
    for chrom, pos, r in rows:
        name = str(r.code) if len(labels) < 2 or r.motif is None else "%s,%s" % (r.code, labels[r.motif])
        head = "\t".join(map(str, (chrom, pos, pos + 1, name, r.cov, r.strand, pos, pos + 1, "255,0,0")))
        out.append(head + "\t" + space.join(map(str, [r.cov, percent(r), r.n_mod, r.n_canon, r.n_other, r.n_delete, r.n_fail, r.n_diff, r.n_nocall])) + "\n")
    return "".join(out)


def partition_files(bam, args):
    """{file name: text} of a --partition-tag run: one file per key, `ungrouped` for reads without any of the tags
    (writers.rs:1045)."""
    out, opts = pileup(bam, args)
    return {("ungrouped" if k is None else k) + ".bed": text(rows, opts) for k, rows in out.items() if rows}


def bedmethyl(bam, args):
    """The bedMethyl text of a run without --partition-tag."""
    out, opts = pileup(bam, args)
    return text(out.get(None, []), opts)
