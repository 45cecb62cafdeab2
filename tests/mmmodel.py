"""An independent model of how `modkit pileup` (reference v0.4.4) reads the MM / ML tags of one record: MM text -> lists ->
forward-read positions -> ML bytes per position, in plain Python, written from the reference's Rust sources:

    parts and headers                MmTagInfo::parse_mm_tag / parse (mod_bam.rs:900-1000)
    delta text                       parse_int_list (mod_bam.rs:881-889) with nom's separated_list1, multispace0, digit1
    deltas -> positions              DeltaListConverter::to_positions[_specific] (mod_bam.rs:697-767)
    ML pointer walk, implicit fill   ModBaseInfo::new / get_base_mod_probs (mod_bam.rs:1213-1295, 1502-1535)
    explicit against inferred        BaseModProbs::combine_checked (mod_bam.rs:629-641)

Its output feeds callmodel.position_maps, so that model and this one together predict every bedMethyl count of a depth-1
read from the record's raw bytes.

Where the reference does not return an error but panics, wraps or (one case) accepts what this project's code representation
cannot hold, the project returns a read error: the read is left out of every count. The model raises ReadError there too.
DESIGN.md section 7 states the same rules.

    case                                                             reference                         here
    delta text of digits that does not fit u32 (any parsed token)    panic (`parse::<u32>().unwrap()`)  ReadError
    `d + n_skips` above u32 (mod_bam.rs:712)                         wraps in a release build           ReadError
    first delta of an N list at or past the read length              panic (index out of bounds)        ReadError
    a header without any code (`C+?`): stride 0                      panic (`chunks(0)`)                ReadError
    a byte >= 0x80 in a header (`split_at` on a character count)     panic or misplaced split           ReadError
    ChEBI code of 2^31 .. 2^32 - 1                                   accepted                           ReadError
    ChEBI text above u32                                             InvalidMm (an error)               ReadError

The ChEBI row is the one place where the project refuses what the reference accepts: a code is held in 32 bits whose top bit
says "ChEBI", so only 31 bits remain for the number (CHEBI_MAX)."""
from callmodel import ReadError

U32_MAX = 0xffffffff
CHEBI_MAX = 0x7fffffff
WS = b" \t\r\n"                     # nom multispace0: space, tab, CR, LF and nothing else (VT and FF are not white space)
DIGITS = b"0123456789"
EXPLICIT, IMPLICIT, DEFAULT = "?", ".", ""


class MmList:
    def __init__(self, base, strand, mode, codes, deltas):
        self.base, self.strand, self.mode, self.codes, self.deltas = base, strand, mode, codes, deltas

    def __repr__(self):
        return "MmList(%r, %r, %r, %r, %r)" % (self.base, self.strand, self.mode, self.codes, self.deltas)

    def __eq__(self, o):
        return (self.base, self.strand, self.mode, self.codes, self.deltas) == (o.base, o.strand, o.mode, o.codes, o.deltas)


def _element(text, i):
    """One element of parse_int_list at text[i:]: multispace0 digit1 multispace0. (value, next index), or None when digit1 fails."""
    while i < len(text) and text[i] in WS:
        i += 1
    j = i
    while j < len(text) and text[j] in DIGITS:
        j += 1
    if j == i:
        return None
    value = int(text[i:j])
    if value > U32_MAX:                                             # mod_bam.rs:885 `num.parse::<u32>().unwrap()`
        raise ReadError("delta does not fit u32")
    while j < len(text) and text[j] in WS:
        j += 1
    return value, j


def parse_int_list(text):
    """separated_list1(tag(","), element): fails when the first element fails; afterwards a separator whose element fails is
    not consumed and the list ends before it. The caller (mod_bam.rs:987) drops whatever text is left."""
    first = _element(text, 0)
    if first is None:
        raise ReadError("invalid MM delta list")
    out, i = [first[0]], first[1]
    while i < len(text) and text[i:i + 1] == b",":
        nxt = _element(text, i + 1)
        if nxt is None:
            break
        out.append(nxt[0])
        i = nxt[1]
    return out


def parse_part(part):
    """MmTagInfo::parse of one `;`-separated part (bytes)."""
    header = part.split(b",")[0]                                    # mod_bam.rs:910-917
    if any(b >= 0x80 for b in header):
        raise ReadError("non-ASCII header")
    h = header.decode("ascii")
    if len(h) < 1 or h[0] not in "ACGTUN":                          # :919-924, FundamentalBase::parse_char
        raise ReadError("fundamental base")
    if len(h) < 2 or h[1] not in "+-":                              # :926-930
        raise ReadError("strand")
    codes, mode, offset, i, seen_chebi = [], None, 2, 2, False
    if i < len(h) and h[i].isdigit():                               # :938-955
        while i < len(h) and h[i].isdigit():
            i += 1
        chebi = int(h[2:i])
        offset += i - 2
        if chebi > CHEBI_MAX:
            raise ReadError("ChEBI code")
        codes.append(chebi)
        seen_chebi = True
    for c in h[i:]:                                                 # :957-982
        if c in "?.":
            mode = EXPLICIT if c == "?" else IMPLICIT
            offset += 1
        elif c.isdigit() or seen_chebi:
            raise ReadError("digit code / ChEBI with letters")
        else:
            codes.append(c)
            offset += 1
    mode = DEFAULT if mode is None else mode                        # :983
    if offset + 1 <= len(part):                                     # :985-997: a comma follows the header
        deltas = parse_int_list(part[offset + 1:])
    else:
        deltas = []
    if not codes:
        raise ReadError("no code: zero stride")
    return MmList(h[0], h[1], mode, codes, deltas)


def parse_mm_tag(mm):
    """parse_mm_tag: split on `;`, drop the empty parts, the first failing part fails the tag (mod_bam.rs:900-907)."""
    return [parse_part(p) for p in mm.split(b";") if p]


def matches(base, nt):                                              # FundamentalBase::matches (mod_bam.rs:858-869)
    return base == "N" or nt == ("T" if base == "U" else base)


def to_positions(base, deltas, fwd):
    """Forward-read positions of a delta list (mod_bam.rs:697-767)."""
    if base == "N":
        if not deltas:
            return []
        pos = [deltas[0]]                                           # the first delta is not checked against the length here
        for d in deltas[1:]:
            nxt = pos[-1] + d + 1
            if nxt >= len(fwd):
                raise ReadError("beyond end of seq")
            pos.append(nxt)
        return pos
    cum, c = [], 0
    for nt in fwd:
        c += matches(base, nt)
        cum.append(c)
    finger, n_skips, out = 0, 0, []
    for d in deltas:
        if finger >= len(cum):
            raise ReadError("beyond end of seq")
        if d + n_skips > U32_MAX:                                   # :712 would wrap
            raise ReadError("u32 wrap")
        while cum[finger] <= d + n_skips:
            finger += 1
            if finger >= len(cum):
                raise ReadError("beyond end of seq")
        out.append(finger)
        n_skips += d + 1
    return out


class Table:
    """One (strand, base) table of a read: `lists` is what callmodel.position_maps takes, [(codes, {position: ML bytes})] in
    MM order; `inferred` {position: [codes]} are the positions an implicit list fills as unmodified; `mode` as
    combine_positions_to_probs leaves it."""

    def __init__(self, mode):
        self.mode, self.lists, self.inferred, self.explicit = mode, [], {}, set()


def mod_base_info(mm, ml, fwd):
    """{(strand, base): Table} of one record: `mm` the MM text (bytes), `ml` the ML bytes, `fwd` the forward read. Raises
    ReadError when the reference would not use the read."""
    tables, pointer = {}, 0
    for L in parse_mm_tag(mm):
        positions = to_positions(L.base, L.deltas, fwd)
        stride = len(L.codes)
        end = pointer + len(L.deltas) * stride
        if end > len(ml):                                           # mod_bam.rs:1222-1228
            raise ReadError("ML array too short")
        per_base = {}
        for k, p in enumerate(positions):                           # :1242-1263
            if p >= len(fwd):
                raise ReadError("first N delta past the end")
            if fwd[p] not in "ACGT":                                # DnaBase::try_from
                raise ReadError("not a DNA base")
            calls, _ = per_base.setdefault(fwd[p], ({}, {}))
            calls[p] = tuple(ml[pointer + k * stride:pointer + (k + 1) * stride])
        if L.mode != EXPLICIT and L.base != "N":                    # :1265-1292 (an N converter has no counts: nothing filled)
            for p, nt in enumerate(fwd):
                if matches(L.base, nt):
                    calls, inferred = per_base.setdefault(nt, ({}, {}))
                    if p not in calls:
                        inferred[p] = list(L.codes)
        for base, (calls, inferred) in per_base.items():            # ModBaseInfo::new :1527-1532, combine_positions_to_probs
            t = tables.get((L.strand, base))
            if t is None:
                t = tables[(L.strand, base)] = Table(L.mode)
            if t.mode != L.mode:
                t.mode = IMPLICIT
            if any(p in t.inferred for p in calls) or any(p in t.explicit for p in inferred):
                raise ReadError("explicit conflicts with inferred")  # combine_checked :630-634
            t.explicit |= set(calls)
            for p, codes in inferred.items():
                t.inferred[p] = t.inferred.get(p, []) + [c for c in codes if c not in t.inferred.get(p, [])]
            if calls:
                t.lists.append((list(L.codes), calls))
        pointer = end                                               # :1534; surplus ML bytes are never looked at
    return tables


def fast_path(text):
    """The documented condition of the kernels' fast tokenizer on a list's delta text: digits and commas only, no empty token,
    at most 9 digits per number."""
    if not text or any(b not in b"0123456789," for b in text):
        return False
    return all(1 <= len(t) <= 9 for t in text.split(b","))
