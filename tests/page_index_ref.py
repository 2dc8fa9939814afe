"""CPU reference for Parquet page indexes -- TEST INFRASTRUCTURE ONLY (imported by tests/ alone).

Reads the ColumnChunk page-index fields of a footer and the ColumnIndex / OffsetIndex structures they point at, with the Thrift reader of
oracle/parquet_oracle.py, and restates from parquet.thrift the row selection that pushed conjuncts leave in a row group: a row leaves
only when the ColumnIndex entry of its page, in the column of some conjunct, proves that conjunct false.  From the selection it derives
what the scan planner must produce: the pages each read column uploads, their covered rows, the segment table that maps selected rows
to covered rows, and the bytes that cross PCIe."""
import math
import struct

from oracle import parquet_oracle as po


def _list(t):
    """list header -> (element type, size)"""
    h = t.b[t.p]
    t.p += 1
    n = h >> 4
    if n == 15:
        n = t.varint()
    return h & 15, n


def _structs(t, n, on_field):
    for _ in range(n):
        t.struct(on_field(t))


def footer_chunks(raw):
    """[[{"oi": (offset, length), "ci": (offset, length), "num_rows"} per column] per row group] from the file footer"""
    flen = struct.unpack_from("<I", raw, len(raw) - 8)[0]
    t = po._T(raw, len(raw) - 8 - flen)
    groups = []

    def chunk_field(cur):
        def f(fid, ty):
            if fid in (4, 5, 6, 7):
                cur[fid] = t.zigzag()
            else:
                t.skip(ty)
        return f

    def rg_field(rg):
        def f(fid, ty):
            if fid == 1:
                _, n = _list(t)
                for _ in range(n):
                    cur = {}
                    t.struct(chunk_field(cur))
                    rg["cols"].append({"oi": (cur.get(4, -1), cur.get(5, 0)), "ci": (cur.get(6, -1), cur.get(7, 0))})
            elif fid == 3:
                rg["num_rows"] = t.zigzag()
            else:
                t.skip(ty)
        return f

    def top(fid, ty):
        if fid == 4:
            _, n = _list(t)
            for _ in range(n):
                rg = {"cols": []}
                t.struct(rg_field(rg))
                for c in rg["cols"]:
                    c["num_rows"] = rg["num_rows"]
                groups.append(rg["cols"])
        else:
            t.skip(ty)
    t.struct(top)
    return groups


def offset_index(raw, pos):
    """OffsetIndex at pos -> [(offset, compressed_page_size, first_row_index)]"""
    t = po._T(raw, pos)
    out = []

    def loc(fid, ty, cur):
        if fid in (1, 2, 3):
            cur[fid] = t.zigzag()
        else:
            t.skip(ty)

    def top(fid, ty):
        if fid == 1:
            _, n = _list(t)
            for _ in range(n):
                cur = {}
                t.struct(lambda f, y: loc(f, y, cur))
                out.append((cur[1], cur[2], cur[3]))
        else:
            t.skip(ty)
    t.struct(top)
    return out


def column_index(raw, pos):
    """ColumnIndex at pos -> {"null_pages": [bool], "min": [bytes], "max": [bytes]}"""
    t = po._T(raw, pos)
    ci = {"null_pages": [], "min": [], "max": []}

    def top(fid, ty):
        if fid == 1:
            _, n = _list(t)
            ci["null_pages"] = [raw[t.p + i] == 1 for i in range(n)]        # a bool in a list is one byte
            t.p += n
        elif fid in (2, 3):
            _, n = _list(t)
            vals = []
            for _ in range(n):
                k = t.varint()
                vals.append(bytes(raw[t.p:t.p + k]))
                t.p += k
            ci["min" if fid == 2 else "max"] = vals
        else:
            t.skip(ty)
    t.struct(top)
    return ci


def page_indexes(raw):
    """[[(offset index or None, column index or None) per column] per row group]"""
    out = []
    for rg in footer_chunks(raw):
        row = []
        for c in rg:
            oi = offset_index(raw, c["oi"][0]) if c["oi"][0] >= 0 and c["oi"][1] > 0 else None
            ci = column_index(raw, c["ci"][0]) if c["ci"][0] >= 0 and c["ci"][1] > 0 else None
            row.append((oi, ci))
        out.append(row)
    return out


def page_rows(oi, num_rows):
    """[(first row, end row)] of every page"""
    return [(oi[i][2], oi[i + 1][2] if i + 1 < len(oi) else num_rows) for i in range(len(oi))]


def stat_value(b, phys):
    if phys == "INT32":
        return struct.unpack("<i", b)[0]
    if phys == "INT64":
        return struct.unpack("<q", b)[0]
    if phys == "FLOAT":
        return struct.unpack("<f", b)[0]
    if phys == "DOUBLE":
        return struct.unpack("<d", b)[0]
    if phys == "FIXED_LEN_BYTE_ARRAY":
        return int.from_bytes(b, "big", signed=True)
    raise ValueError(phys)


def excludes(op, lit, mn, mx, all_null):
    """True = no row with these statistics satisfies `column op lit` (op: eq lt le gt ge notnull)"""
    if all_null:
        return True
    if op == "notnull" or mn is None or mx is None:
        return False
    if isinstance(mn, float) and (math.isnan(mn) or math.isnan(mx)):
        return False
    return {"eq": lit < mn or lit > mx, "lt": not mn < lit, "le": not mn <= lit, "gt": not mx > lit, "ge": not mx >= lit}[op]


def selection(terms, indexes, num_rows):
    """terms: [(column position, op, literal, physical type)]; indexes: [(offset index, column index)] per column.
    -> sorted disjoint [begin, end) ranges of the rows no term's page statistics rule out"""
    out = []
    for col, op, lit, phys in terms:
        oi, ci = indexes[col]
        for i, (a, b) in enumerate(page_rows(oi, num_rows)):
            null = ci["null_pages"][i]
            mn = None if null else stat_value(ci["min"][i], phys)
            mx = None if null else stat_value(ci["max"][i], phys)
            if excludes(op, lit, mn, mx, null):
                out.append((a, b))
    ranges, at = [], 0
    for a, b in sorted(out):
        if a > at:
            ranges.append((at, a))
        at = max(at, b)
    if at < num_rows:
        ranges.append((at, num_rows))
    return ranges


def column_window(oi, num_rows, ranges):
    """-> (selected page indices, covered rows, [(out_row, cov_row, count)] one per range)"""
    pages, cov_at, covered = [], {}, 0
    spans = page_rows(oi, num_rows)
    for i, (a, b) in enumerate(spans):
        if any(ra < b and a < rb for ra, rb in ranges):
            pages.append(i)
            cov_at[i] = covered
            covered += b - a
    segs, out = [], 0
    for ra, rb in ranges:
        i = next(k for k, (a, b) in enumerate(spans) if a <= ra < b)
        segs.append((out, cov_at[i] + ra - spans[i][0], rb - ra))
        out += rb - ra
    return pages, covered, segs


def chunk_pieces(start, oi, pages):
    """file byte ranges a page-pruned chunk uploads: the bytes before its first data page, then each run of selected pages"""
    out = [[start, oi[0][0]]] if oi[0][0] > start else []
    prev = None
    for i in pages:
        off, size, _ = oi[i]
        if prev is not None and i == prev + 1 and out[-1][1] == off:
            out[-1][1] = off + size
        else:
            out.append([off, off + size])
        prev = i
    return out


def upload_bytes(items):
    """bytes of the upload ranges over one unit's [start, end) items: sorted, a gap of up to 64 KB rides along"""
    total, cur = 0, None
    for a, b in sorted(items):
        if cur is not None and a - cur[1] <= 65536:
            cur[1] = max(cur[1], b)
        else:
            if cur is not None:
                total += cur[1] - cur[0]
            cur = [a, b]
    return total + (cur[1] - cur[0] if cur else 0)
