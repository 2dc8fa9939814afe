"""A Parquet writer for tests that builds every byte by hand, restated from parquet-format `parquet.thrift` (Thrift compact protocol),
`Encodings.md` (PLAIN, RLE / bit-packed hybrid) and google/snappy `format_description.txt`.

Stock writers emit a narrow subset of legal Parquet: RLE runs of 8 or more repeats only, minimal bit widths, Snappy streams cut into
independent 64 KiB fragments.  Here each layer takes an explicit shape instead -- the run list of a hybrid stream, the element list of
a Snappy stream, each page's version, encoding, codec and level layout -- so the decoders' other branches can be reached.  Every file
comes with the values and validity it is meant to hold: `Chunk.values` / `Chunk.valid`, the tests' expected output.

Flat columns only."""
import struct

import numpy as np

# parquet.thrift enums
INT32, INT64, FLOAT, DOUBLE, BYTE_ARRAY, FLBA = 1, 2, 4, 5, 6, 7
PLAIN, PLAIN_DICTIONARY, RLE, BIT_PACKED, RLE_DICTIONARY = 0, 2, 3, 4, 8
NONE, SNAPPY, ZSTD = 0, 1, 6
DATA_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 2, 3
CT_DECIMAL, CT_DATE, CT_INT_8, CT_INT_16 = 5, 6, 15, 16


# ---- Thrift compact protocol ---------------------------------------------------------------------------------------------------
_BOOL, _I32, _I64, _BIN, _LIST, _STRUCT = 1, 5, 6, 8, 9, 12


def uleb(n):
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | (0x80 if n else 0))
        if not n:
            return bytes(out)


def _zz(n):
    return (n << 1) ^ (n >> 63)


def _value(kind, v):
    if kind in (_I32, _I64):
        return uleb(_zz(v))
    if kind == _BIN:
        b = v.encode() if isinstance(v, str) else bytes(v)
        return uleb(len(b)) + b
    if kind == _STRUCT:
        return _struct(v)
    et, items = v                                                    # _LIST
    head = bytes([(len(items) << 4) | et]) if len(items) < 15 else bytes([0xF0 | et]) + uleb(len(items))
    return head + b"".join(_value(et, x) for x in items)


def _struct(fields):
    """fields: [(field id, kind, value)] in increasing field id; None values are left out"""
    out, last = bytearray(), 0
    for fid, kind, v in fields:
        if v is None:
            continue
        t = (1 if v else 2) if kind == _BOOL else kind
        d = fid - last
        out += bytes([(d << 4) | t]) if 0 < d <= 15 else bytes([t]) + uleb(_zz(fid))
        last = fid
        if kind != _BOOL:
            out += _value(kind, v)
    out.append(0)
    return bytes(out)


# ---- RLE / bit-packed hybrid ---------------------------------------------------------------------------------------------------
def pack_bits(values, bit_width):
    """values LSB first, bit_width bits each"""
    acc = nbits = 0
    out = bytearray()
    for v in values:
        acc |= (int(v) & ((1 << bit_width) - 1)) << nbits
        nbits += bit_width
        while nbits >= 8:
            out.append(acc & 0xFF)
            acc >>= 8
            nbits -= 8
    if nbits:
        out.append(acc & 0xFF)
    return bytes(out)


def hybrid(runs, bit_width):
    """runs: ("rle", count, value) | ("packed", groups, values) -- values padded with zeros to groups x 8 -- | ("raw", bytes).  An
    optional last element of an "rle" / "packed" run is the header's ULEB128 length in bytes (a longer, non-minimal encoding)."""
    out = bytearray()
    vbytes = (bit_width + 7) // 8
    for r in runs:
        if r[0] == "raw":
            out += r[1]
            continue
        h = (r[1] << 1) | (r[0] == "packed")
        head = uleb(h)
        if len(r) > 3 and r[3] > len(head):
            head = bytes(b | 0x80 for b in head) + b"\x80" * (r[3] - len(head) - 1) + b"\x00"
        out += head
        if r[0] == "rle":
            out += int(r[2]).to_bytes(vbytes, "little")
        else:
            vals = list(r[2]) + [0] * (r[1] * 8 - len(r[2]))
            out += pack_bits(vals, bit_width)
    return bytes(out)


def runs_of(values, shape):
    """A run list that encodes `values` in the given shape:
    packed       one bit-packed run (the last group padded past the values)
    rle          every maximal stretch of equal values an RLE run, however short
    rle1         an RLE run of 1 per value: the most runs a stream can hold
    mixed        8 values bit-packed, then the next 1 to 7 values as RLE runs of 1, alternating
    zero_runs    mixed, with a zero-length run of either kind after every run (Arrow's reader takes one for the end of the stream)
    long_tail    like rle, but the final RLE run claims more values than are left
    packed_runs  bit-packed runs of 1 to 3 groups, two-byte headers on every other run"""
    values = [int(v) for v in values]
    n = len(values)
    if shape == "packed":
        return [("packed", (n + 7) // 8, values)] if n else []
    if shape in ("rle", "rle1", "long_tail"):
        runs, i = [], 0
        while i < n:
            j = i + 1
            if shape != "rle1":
                while j < n and values[j] == values[i]:
                    j += 1
            runs.append(("rle", j - i, values[i]))
            i = j
        if shape == "long_tail" and runs:
            runs[-1] = ("rle", runs[-1][1] + 13, runs[-1][2])
        return runs
    if shape in ("mixed", "zero_runs"):
        zero = shape == "zero_runs"
        runs, i, k = [], 0, 0
        while i < n:
            if k % 2 == 0:
                runs.append(("packed", 1, values[i:i + 8]))
                i += 8
                runs += [("rle", 0, 0)] if zero else []
            else:
                j = min(n, i + 1 + k % 7)
                for v in values[i:j]:
                    runs.append(("rle", 1, v))
                i = j
                runs += [("packed", 0, [])] if zero else []
            k += 1
        return runs
    if shape == "packed_runs":
        runs, i, k = [], 0, 0
        while i < n:
            g = 1 + k % 3
            runs.append(("packed", g, values[i:i + 8 * g], 2 if k % 2 else 1))
            i += 8 * g
            k += 1
        return runs
    raise ValueError(shape)


# ---- Snappy (format_description.txt) -------------------------------------------------------------------------------------------
def sn_literal(data, form=None):
    """form: None = the shortest; 0 = length in the tag (1..60 bytes); 1..4 = length in that many extra bytes"""
    n = len(data) - 1
    if form is None:
        form = 0 if n < 60 else (n.bit_length() + 7) // 8
    if form == 0:
        assert n < 60
        return bytes([n << 2]) + bytes(data)
    assert n < 1 << (8 * form)
    return bytes([(59 + form) << 2]) + n.to_bytes(form, "little") + bytes(data)


def sn_copy(offset, length, kind=None):
    """kind 1: 4..11 bytes at offsets < 2048; 2: 1..64 bytes at offsets < 65536; 4: 1..64 bytes at any offset"""
    if kind is None:
        kind = 1 if 4 <= length <= 11 and offset < 2048 else 2 if offset < 65536 else 4
    if kind == 1:
        assert 4 <= length <= 11 and 0 < offset < 2048
        return bytes([((offset >> 8) << 5) | ((length - 4) << 2) | 1, offset & 0xFF])
    assert 1 <= length <= 64
    if kind == 2:
        return bytes([((length - 1) << 2) | 2]) + offset.to_bytes(2, "little")
    return bytes([((length - 1) << 2) | 3]) + offset.to_bytes(4, "little")


def snappy(elements):
    """elements: ("lit", bytes[, form]) | ("copy", offset, length[, kind]).  -> (stream, the bytes it decodes to)"""
    body, out = bytearray(), bytearray()
    for e in elements:
        if e[0] == "lit":
            body += sn_literal(e[1], e[2] if len(e) > 2 else None)
            out += e[1]
        else:
            off, ln = e[1], e[2]
            body += sn_copy(off, ln, e[3] if len(e) > 3 else None)
            for _ in range(ln):
                out.append(out[-off])
    return uleb(len(out)) + bytes(body), bytes(out)


def snappy_elements(data, copy_kind=None, lit_form=None, max_lit=1 << 20, window=1 << 20, min_match=4):
    """A greedy element list for `data`: 4-byte matches found through a hash of the last position of every 4-byte prefix, copies of at
    most 64 bytes (of `copy_kind`, when it can say the match), literals of at most max_lit bytes (in lit_form when it fits)."""
    data = bytes(data)
    n, last, els, lit0, i = len(data), {}, [], 0, 0

    def flush(end):
        s = lit0
        while s < end:
            e = min(end, s + max_lit)
            form = lit_form if lit_form is not None and (lit_form > 0 or e - s <= 60) and (lit_form == 0 or e - s - 1 < 1 << (8 * lit_form)) else None
            els.append(("lit", data[s:e]) + ((form,) if form is not None else ()))
            s = e
    while i + min_match <= n:
        key = data[i:i + 4]
        j = last.get(key)
        last[key] = i
        if j is not None and i - j <= window and (copy_kind != 1 or i - j < 2048):
            ln = 4
            while i + ln < n and ln < 64 and data[j + ln] == data[i + ln]:
                ln += 1
            if copy_kind == 1:
                ln = min(ln, 11)
            if copy_kind == 2 and i - j >= 65536:
                i += 1
                continue
            flush(i)
            els.append(("copy", i - j, ln) + ((copy_kind,) if copy_kind else ()))
            i += ln
            lit0 = i
        else:
            i += 1
    lit0 = min(lit0, n)
    flush(n)
    return els


# ---- PLAIN values --------------------------------------------------------------------------------------------------------------
def plain(phys, values, type_length=0):
    """values: ints (INT32 / INT64 / FLBA, FLOAT / DOUBLE as their bit patterns) or bytes (BYTE_ARRAY)"""
    if phys in (INT32, FLOAT):
        return np.asarray([int(v) & 0xFFFFFFFF for v in values], dtype="<u4").tobytes()
    if phys in (INT64, DOUBLE):
        return np.asarray([int(v) & (2**64 - 1) for v in values], dtype="<u8").tobytes()
    if phys == FLBA:
        return b"".join(int(v).to_bytes(type_length, "big", signed=True) for v in values)
    if phys == BYTE_ARRAY:
        return b"".join(struct.pack("<I", len(v)) + bytes(v) for v in values)
    raise ValueError(phys)


# ---- pages, chunks, files ------------------------------------------------------------------------------------------------------
class Page:
    """One page as stored: kind DATA_PAGE / DATA_PAGE_V2 / DICTIONARY_PAGE.  v1: `body` = [u32 level length][levels][values] (levels
    present for optional columns); v2: `levels` + `body` = the values section."""

    def __init__(self, kind, num_values, encoding, body, levels=b"", num_nulls=0, def_encoding=RLE, compressed=True, elements=None):
        self.kind, self.num_values, self.encoding, self.body, self.levels = kind, num_values, encoding, bytes(body), bytes(levels)
        self.num_nulls, self.def_encoding, self.compressed, self.elements = num_nulls, def_encoding, compressed, elements

    def encode(self, codec):
        """-> header + stored bytes.  elements: a Snappy element list for the compressed section (codec SNAPPY)"""
        compress = codec != NONE and (self.kind != DATA_PAGE_V2 or self.compressed)
        if not compress:
            stored = self.body
        elif codec == SNAPPY:
            stream, got = snappy(self.elements if self.elements is not None else snappy_elements(self.body))
            assert got == self.body
            stored = stream
        else:
            import pyarrow as pa
            stored = pa.compress(self.body, codec="zstd", asbytes=True)
        stored = self.levels + stored
        unc = len(self.levels) + len(self.body)
        if self.kind == DICTIONARY_PAGE:
            sub = (7, _STRUCT, [(1, _I32, self.num_values), (2, _I32, self.encoding)])
        elif self.kind == DATA_PAGE:
            sub = (5, _STRUCT, [(1, _I32, self.num_values), (2, _I32, self.encoding), (3, _I32, self.def_encoding), (4, _I32, RLE)])
        else:
            sub = (8, _STRUCT, [(1, _I32, self.num_values), (2, _I32, self.num_nulls), (3, _I32, self.num_values), (4, _I32, self.encoding),
                                (5, _I32, len(self.levels)), (6, _I32, 0), (7, _BOOL, bool(self.compressed))])
        header = _struct([(1, _I32, self.kind), (2, _I32, unc), (3, _I32, len(stored)), sub])
        return header + stored


class Column:
    """A flat column of the schema.  phys: INT32 / INT64 / FLOAT / DOUBLE / FLBA / BYTE_ARRAY; converted: parquet ConvertedType"""

    def __init__(self, name, phys, optional=True, type_length=0, converted=None, precision=0, scale=0):
        self.name, self.phys, self.optional, self.type_length = name, phys, optional, type_length
        self.converted, self.precision, self.scale = converted, precision, scale

    def schema_element(self):
        dec = self.converted == CT_DECIMAL
        return [(1, _I32, self.phys), (2, _I32, self.type_length or None), (3, _I32, 1 if self.optional else 0), (4, _BIN, self.name),
                (6, _I32, self.converted), (7, _I32, self.scale if dec else None), (8, _I32, self.precision if dec else None)]


class Chunk:
    """One column chunk: its pages (a dictionary page first, if any) and what they hold.  null_count: the Statistics value written to
    the footer (None: no Statistics)."""

    def __init__(self, pages, values, valid, codec=NONE, null_count=None):
        self.pages, self.values, self.valid, self.codec, self.null_count = pages, list(values), list(valid), codec, null_count
        assert len(self.values) == len(self.valid) == sum(p.num_values for p in pages if p.kind != DICTIONARY_PAGE)


def write_file(columns, row_groups):
    """columns: [Column]; row_groups: [[Chunk per column]].  -> the file's bytes"""
    out = bytearray(b"PAR1")
    rgs, total_rows = [], 0
    for chunks in row_groups:
        rows = len(chunks[0].values)
        assert all(len(c.values) == rows for c in chunks)
        ccs = []
        for col, ch in zip(columns, chunks):
            start = len(out)
            dict_off = data_off = None
            encs = {RLE}
            for p in ch.pages:
                if p.kind == DICTIONARY_PAGE:
                    dict_off = len(out)
                elif data_off is None:
                    data_off = len(out)
                encs.add(p.encoding)
                out += p.encode(ch.codec)
            size = len(out) - start
            stats = None if ch.null_count is None else [(3, _I64, ch.null_count)]
            meta = [(1, _I32, col.phys), (2, _LIST, (_I32, sorted(encs))), (3, _LIST, (_BIN, [col.name])), (4, _I32, ch.codec), (5, _I64, rows),
                    (6, _I64, size), (7, _I64, size), (9, _I64, data_off if data_off is not None else start), (11, _I64, dict_off),
                    (12, _STRUCT, stats)]
            ccs.append([(2, _I64, start), (3, _STRUCT, meta)])
        rgs.append([(1, _LIST, (_STRUCT, ccs)), (2, _I64, 0), (3, _I64, rows)])
        total_rows += rows
    schema = [[(4, _BIN, "schema"), (5, _I32, len(columns))]] + [c.schema_element() for c in columns]
    footer = _struct([(1, _I32, 1), (2, _LIST, (_STRUCT, schema)), (3, _I64, total_rows), (4, _LIST, (_STRUCT, rgs)), (6, _BIN, "pqwrite")])
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    return bytes(out)


# ---- chunks from values --------------------------------------------------------------------------------------------------------
def data_page(col, values, valid, version=1, encoding=PLAIN, dictionary=None, bit_width=None, index_shape="rle", level_shape="rle",
              compressed=True):
    """One data page holding values[k] at the rows where valid[k] (values of NULL rows are ignored).  Dictionary encodings: `dictionary`
    lists the page's dictionary; the indices are written at `bit_width` (default: the least that holds them) in `index_shape`."""
    valid = [bool(v) for v in valid]
    present = [v for v, ok in zip(values, valid) if ok]
    if encoding in (PLAIN_DICTIONARY, RLE_DICTIONARY):
        pos = {}
        for k, v in enumerate(dictionary):
            pos.setdefault(v, k)
        idx = [pos[v] for v in present]
        bw = bit_width if bit_width is not None else max(len(dictionary) - 1, 0).bit_length()
        vals = bytes([bw]) + hybrid(runs_of(idx, index_shape), bw)
    else:
        vals = plain(col.phys, present, col.type_length)
    levels = hybrid(runs_of([int(v) for v in valid], level_shape), 1) if col.optional else b""
    n, nulls = len(valid), valid.count(False)
    if version == 1:
        body = (struct.pack("<I", len(levels)) + levels if col.optional else b"") + vals
        return Page(DATA_PAGE, n, encoding, body)
    return Page(DATA_PAGE_V2, n, encoding, vals, levels=levels, num_nulls=nulls, compressed=compressed)


def dict_page(col, dictionary):
    return Page(DICTIONARY_PAGE, len(dictionary), PLAIN_DICTIONARY, plain(col.phys, dictionary, col.type_length))


def chunk(col, values, valid, page_rows, codec=NONE, null_count="exact", dictionary=None, fallback_at=None, **page_kw):
    """values / valid split into pages of page_rows rows (a list: one size per page, cycled).  dictionary: every page dictionary-encoded
    against it, except pages starting at or after row `fallback_at`, which fall back to PLAIN.  null_count: "exact", None (no Statistics)
    or an int written as is."""
    valid = [bool(v) for v in valid]
    sizes = page_rows if isinstance(page_rows, (list, tuple)) else [page_rows]
    pages = [dict_page(col, dictionary)] if dictionary is not None else []
    r, k = 0, 0
    n = len(values)
    while r < n or (n == 0 and k == 0):
        m = sizes[k % len(sizes)]
        end = min(n, r + m)
        dict_enc = dictionary is not None and (fallback_at is None or r < fallback_at)
        kw = dict(page_kw)
        if dict_enc:
            kw.setdefault("encoding", RLE_DICTIONARY)
        else:
            kw["encoding"] = PLAIN
        pages.append(data_page(col, values[r:end], valid[r:end], dictionary=dictionary if dict_enc else None, **kw))
        r, k = end, k + 1
        if n == 0:
            break
    nc = valid.count(False) if null_count == "exact" else null_count
    return Chunk(pages, values, valid, codec, nc)
