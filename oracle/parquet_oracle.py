"""CPU restatement of Parquet column-chunk decode -- TEST INFRASTRUCTURE ONLY (imported by tests/ alone).

The reference reaches the third-party `parquet` crate 58.4.0 for this step (native/core/src/parquet/parquet_exec.rs:139-141,
features `snap,lz4,zstd,flate2` native/core/Cargo.toml:40); its source is not under /root/reference, so the decode is restated
from the published format: parquet-format `parquet.thrift` (PageHeader), `Encodings.md` (PLAIN, RLE/bit-packed hybrid,
RLE_DICTIONARY), `Compression.md` (SNAPPY = raw snappy block) and google/snappy `format_description.txt`.
Parity status: pinned on CPU against pyarrow's reader (Arrow C++, an independent implementation) over the same files the GPU
tests use (tests/test_parquet_cpu.py); NOT pinned against the reference itself (cannot be built here).

Scope = what the device decoder covers: flat columns, data pages v1 / v2, UNCOMPRESSED / SNAPPY / ZSTD (through pyarrow), PLAIN and dictionary
encodings, INT32 / INT64 / FLOAT / DOUBLE / FIXED_LEN_BYTE_ARRAY (decimals) / BYTE_ARRAY (dictionary strings)."""
import struct

import numpy as np


# ---- Thrift compact protocol: just enough for PageHeader -----------------------------------------------------------------
class _T:
    def __init__(self, buf, pos):
        self.b, self.p = buf, pos

    def varint(self):
        r = s = 0
        while True:
            c = self.b[self.p]
            self.p += 1
            r |= (c & 0x7F) << s
            s += 7
            if not c & 0x80:
                return r

    def zigzag(self):
        v = self.varint()
        return (v >> 1) ^ -(v & 1)

    def skip(self, t):
        if t in (1, 2):
            return
        if t == 3:
            self.p += 1
        elif t in (4, 5, 6):
            self.varint()
        elif t == 7:
            self.p += 8
        elif t == 8:
            n = self.varint()
            self.p += n
        elif t in (9, 10):
            h = self.b[self.p]
            self.p += 1
            n = h >> 4
            if n == 15:
                n = self.varint()
            for _ in range(n):
                self.skip(h & 15)
        elif t == 12:
            self.struct(lambda fid, ty: self.skip(ty))
        else:
            raise ValueError(f"thrift type {t}")

    def struct(self, on_field):
        last = 0
        while True:
            h = self.b[self.p]
            self.p += 1
            if h == 0:
                return
            ty, delta = h & 15, h >> 4
            fid = last + delta if delta else self.zigzag()
            last = fid
            on_field(fid, ty)


def page_header(buf, pos):
    """-> (dict, position of the first byte after the header)"""
    t = _T(buf, pos)
    h = {"type": None, "uncompressed": 0, "compressed": 0, "num_values": 0, "encoding": 0, "def_encoding": 3, "def_bytes": 0, "rep_bytes": 0,
         "v2_compressed": True}

    def sub(fields):
        def f(fid, ty):
            if fid in fields:
                name = fields[fid]
                h[name] = (ty == 1) if name == "v2_compressed" else t.zigzag()
            else:
                t.skip(ty)
        return f

    def top(fid, ty):
        if fid == 1:
            h["type"] = t.zigzag()
        elif fid == 2:
            h["uncompressed"] = t.zigzag()
        elif fid == 3:
            h["compressed"] = t.zigzag()
        elif fid == 5:
            t.struct(sub({1: "num_values", 2: "encoding", 3: "def_encoding"}))
        elif fid == 7:
            t.struct(sub({1: "num_values", 2: "encoding"}))
        elif fid == 8:
            t.struct(sub({1: "num_values", 4: "encoding", 5: "def_bytes", 6: "rep_bytes", 7: "v2_compressed"}))
        else:
            t.skip(ty)
    t.struct(top)
    return h, t.p


# ---- Snappy raw block (format_description.txt) ---------------------------------------------------------------------------
def snappy_decompress(src):
    src = bytes(src)
    n = shift = pos = 0
    while True:
        c = src[pos]
        pos += 1
        n |= (c & 0x7F) << shift
        shift += 7
        if not c & 0x80:
            break
    out = bytearray()
    while pos < len(src):
        tag = src[pos]
        pos += 1
        t = tag & 3
        if t == 0:
            ln = tag >> 2
            if ln >= 60:
                extra = ln - 59
                ln = int.from_bytes(src[pos:pos + extra], "little")
                pos += extra
            ln += 1
            out += src[pos:pos + ln]
            pos += ln
            continue
        if t == 1:
            ln, off = ((tag >> 2) & 7) + 4, ((tag >> 5) << 8) | src[pos]
            pos += 1
        elif t == 2:
            ln, off = (tag >> 2) + 1, int.from_bytes(src[pos:pos + 2], "little")
            pos += 2
        else:
            ln, off = (tag >> 2) + 1, int.from_bytes(src[pos:pos + 4], "little")
            pos += 4
        assert 0 < off <= len(out)
        for _ in range(ln):                      # byte-wise: copies may overlap their own output
            out.append(out[-off])
    assert len(out) == n
    return bytes(out)


# ---- RLE / bit-packed hybrid (Encodings.md) ------------------------------------------------------------------------------
def rle_hybrid(buf, bit_width, count):
    out = np.zeros(count, dtype=np.int64)
    pos = got = 0
    vbytes = (bit_width + 7) // 8
    while got < count and pos < len(buf):
        h = shift = 0
        while True:
            c = buf[pos]
            pos += 1
            h |= (c & 0x7F) << shift
            shift += 7
            if not c & 0x80:
                break
        if h & 1:
            groups = h >> 1
            nbytes = groups * bit_width
            bits = np.unpackbits(np.frombuffer(buf[pos:pos + nbytes], dtype=np.uint8), bitorder="little")
            vals = bits[: groups * 8 * bit_width].reshape(-1, bit_width).astype(np.int64) @ (1 << np.arange(bit_width, dtype=np.int64)) if bit_width else np.zeros(groups * 8, dtype=np.int64)
            take = min(count - got, groups * 8)
            out[got:got + take] = vals[:take]
            got += take
            pos += nbytes
        else:
            run = h >> 1
            v = int.from_bytes(buf[pos:pos + vbytes], "little")
            pos += vbytes
            take = min(count - got, run)
            out[got:got + take] = v
            got += take
    assert got == count, "hybrid stream shorter than the page's value count"
    return out


# ---- PLAIN ---------------------------------------------------------------------------------------------------------------
def plain(buf, phys, n, type_length=0):
    if phys == "INT32":
        return np.frombuffer(buf[:4 * n], dtype="<i4").astype(np.int64)
    if phys == "INT64":
        return np.frombuffer(buf[:8 * n], dtype="<i8")
    if phys == "FLOAT":
        return np.frombuffer(buf[:4 * n], dtype="<f4")
    if phys == "DOUBLE":
        return np.frombuffer(buf[:8 * n], dtype="<f8")
    if phys == "FIXED_LEN_BYTE_ARRAY":                      # big-endian two's complement (decimals): python ints
        return np.array([int.from_bytes(buf[i * type_length:(i + 1) * type_length], "big", signed=True) for i in range(n)], dtype=object)
    if phys == "BYTE_ARRAY":
        out, pos = [], 0
        for _ in range(n):
            (ln,) = struct.unpack_from("<I", buf, pos)
            out.append(bytes(buf[pos + 4:pos + 4 + ln]))
            pos += 4 + ln
        return np.array(out, dtype=object)
    raise ValueError(phys)


def _decompress(codec, raw, n):
    if codec == "SNAPPY":
        return snappy_decompress(raw)
    if codec == "ZSTD":                                                          # Compression.md: a zstd frame; not restated here
        import pyarrow as pa
        return pa.decompress(raw, n, codec="zstd", asbytes=True)
    assert codec == "UNCOMPRESSED", codec
    return raw


# ---- one column chunk ----------------------------------------------------------------------------------------------------
def decode_chunk(file_bytes, start, total_compressed, num_values, phys, codec, optional, type_length=0):
    """-> (values as a numpy array with None-equivalent 0 at NULL rows, valid bool array).  `start` = dictionary_page_offset or
    data_page_offset, whichever comes first (ColumnMetaData)."""
    pos, end = start, start + total_compressed
    dictionary = None
    vals, valid = [], []
    seen = 0
    while pos < end and seen < num_values:
        h, body = page_header(file_bytes, pos)
        raw = file_bytes[body:body + h["compressed"]]
        pos = body + h["compressed"]
        if h["type"] == 2:                                                       # DICTIONARY_PAGE
            data = _decompress(codec, raw, h["uncompressed"])
            dictionary = plain(data, phys, h["num_values"], type_length)
            continue
        if h["type"] not in (0, 3):
            continue
        n = h["num_values"]
        if h["type"] == 0:                                                       # v1: levels inside the compressed body
            data = _decompress(codec, raw, h["uncompressed"])
            if optional:
                assert h["def_encoding"] == 3, "definition levels other than RLE (BIT_PACKED) are refused"
                (dl,) = struct.unpack_from("<I", data, 0)
                levels = rle_hybrid(data[4:4 + dl], 1, n)
                data = data[4 + dl:]
            else:
                levels = np.ones(n, dtype=np.int64)
        else:                                                                    # v2: levels uncompressed, in front
            lv = h["rep_bytes"] + h["def_bytes"]
            assert not (optional and n and not h["def_bytes"]), "data page v2 of an optional column without definition levels"
            levels = rle_hybrid(raw[h["rep_bytes"]:lv], 1, n) if optional else np.ones(n, dtype=np.int64)
            data = raw[lv:]
            if h["v2_compressed"]:
                data = _decompress(codec, data, h["uncompressed"] - lv)
        nn = int(levels.sum())
        if h["encoding"] == 0:
            dense = plain(data, phys, nn, type_length)
        elif h["encoding"] in (2, 8):
            idx = rle_hybrid(data[1:], data[0], nn)
            dense = dictionary[idx]
        else:
            raise ValueError(f"encoding {h['encoding']}")
        page_vals = np.zeros(n, dtype=dense.dtype if dense.dtype != object else object)
        ok = levels.astype(bool)
        page_vals[ok] = dense
        vals.append(page_vals)
        valid.append(ok)
        seen += n
    return np.concatenate(vals), np.concatenate(valid)
