"""CPU restatement of the Parquet value encodings DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and BYTE_STREAM_SPLIT
(parquet-format `Encodings.md`) -- test infrastructure, imported by tests/ alone.

Page headers, Snappy, the RLE/bit-packed hybrid and PLAIN come from oracle/parquet_oracle.py; decode_chunk() below walks a column
chunk like that module's decode_chunk() and adds these four encodings to PLAIN and dictionary pages.  Pinned against pyarrow's reader
in tests/test_parquet_encodings_cpu.py."""
import struct

import numpy as np

from oracle import parquet_oracle as po


def uleb(buf, pos):
    """-> (ULEB128 value at buf[pos], position after it)"""
    r = s = 0
    while True:
        c = buf[pos]
        pos += 1
        r |= (c & 0x7F) << s
        s += 7
        if not c & 0x80:
            return r, pos


def delta_binary_packed(buf, bits=64, pos=0):
    """-> (python ints, position after the stream).  Values wrap in `bits` (two's complement)."""
    block, pos = uleb(buf, pos)
    mbs, pos = uleb(buf, pos)
    total, pos = uleb(buf, pos)
    z, pos = uleb(buf, pos)
    per_mb = block // mbs
    assert block % 128 == 0 and per_mb % 32 == 0
    mod = 1 << bits
    wrap = lambda v: ((v + (mod >> 1)) % mod) - (mod >> 1)
    out = [wrap((z >> 1) ^ -(z & 1))] if total else []
    while len(out) < total:
        z, pos = uleb(buf, pos)
        min_delta = (z >> 1) ^ -(z & 1)
        widths = buf[pos:pos + mbs]
        pos += mbs
        for bw in widths:
            if len(out) >= total:
                break                                   # unused miniblocks: any width, no body bytes
            assert bw <= bits
            body = int.from_bytes(buf[pos:pos + per_mb * bw // 8], "little")
            pos += per_mb * bw // 8
            for k in range(min(per_mb, total - len(out))):
                out.append(wrap(out[-1] + min_delta + ((body >> (k * bw)) & ((1 << bw) - 1))))
    return out, pos


def delta_length_byte_array(buf, pos=0):
    """-> (list of bytes, position after the section)"""
    lens, pos = delta_binary_packed(buf, 32, pos)
    out = []
    for ln in lens:
        out.append(bytes(buf[pos:pos + ln]))
        pos += ln
    return out, pos


def delta_byte_array(buf):
    prefix, pos = delta_binary_packed(buf, 32, 0)
    suffix, _ = delta_length_byte_array(buf, pos)
    out, prev = [], b""
    for p, s in zip(prefix, suffix):
        prev = prev[:p] + s
        out.append(prev)
    return out


def byte_stream_split(buf, phys, n, type_length=0):
    w = {"INT32": 4, "FLOAT": 4, "INT64": 8, "DOUBLE": 8}.get(phys, type_length)
    assert len(buf) >= w * n
    joined = np.frombuffer(bytes(buf[:w * n]), dtype=np.uint8).reshape(w, n).T.copy().tobytes()  # byte k of value i at [k * n + i]
    return po.plain(joined, phys, n, type_length)


def values(data, encoding, phys, nn, dictionary, type_length=0):
    """the `nn` non-null values of one page's values section"""
    if encoding == 0:
        return po.plain(data, phys, nn, type_length)
    if encoding in (2, 8):
        return dictionary[po.rle_hybrid(data[1:], data[0], nn)]
    if encoding == 5:                                                        # DELTA_BINARY_PACKED (INT32 / INT64)
        v, _ = delta_binary_packed(data, 32 if phys == "INT32" else 64)
        assert len(v) == nn
        return np.array(v, dtype=np.int64)
    if encoding in (6, 7):                                                   # DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY
        raw = delta_length_byte_array(data)[0] if encoding == 6 else delta_byte_array(data)
        assert len(raw) == nn
        if phys == "FIXED_LEN_BYTE_ARRAY":
            return np.array([int.from_bytes(v, "big", signed=True) for v in raw], dtype=object)
        return np.array(raw, dtype=object)
    if encoding == 9:                                                        # BYTE_STREAM_SPLIT
        return byte_stream_split(data, phys, nn, type_length)
    raise ValueError(f"encoding {encoding}")


def decode_chunk(file_bytes, start, total_compressed, num_values, phys, codec, optional, type_length=0):
    """-> (values with 0 at NULL rows, valid bool array) of a column chunk; UNCOMPRESSED / SNAPPY, data pages v1 / v2"""
    pos, end = start, start + total_compressed
    dictionary = None
    vals, valid = [], []
    seen = 0
    while pos < end and seen < num_values:
        h, body = po.page_header(file_bytes, pos)
        raw = file_bytes[body:body + h["compressed"]]
        pos = body + h["compressed"]
        if h["type"] == 2:
            data = po.snappy_decompress(raw) if codec == "SNAPPY" else raw
            dictionary = po.plain(data, phys, h["num_values"], type_length)
            continue
        if h["type"] not in (0, 3):
            continue
        n = h["num_values"]
        if h["type"] == 0:
            data = po.snappy_decompress(raw) if codec == "SNAPPY" else raw
            if optional:
                (dl,) = struct.unpack_from("<I", data, 0)
                levels = po.rle_hybrid(data[4:4 + dl], 1, n)
                data = data[4 + dl:]
            else:
                levels = np.ones(n, dtype=np.int64)
        else:
            lv = h["rep_bytes"] + h["def_bytes"]
            levels = po.rle_hybrid(raw[h["rep_bytes"]:lv], 1, n) if optional and h["def_bytes"] else np.ones(n, dtype=np.int64)
            data = raw[lv:]
            if codec == "SNAPPY" and h["v2_compressed"]:
                data = po.snappy_decompress(data)
        dense = values(data, h["encoding"], phys, int(levels.sum()), dictionary, type_length)
        page_vals = np.zeros(n, dtype=dense.dtype if dense.dtype != object else object)
        ok = levels.astype(bool)
        page_vals[ok] = dense
        vals.append(page_vals)
        valid.append(ok)
        seen += n
    return np.concatenate(vals), np.concatenate(valid)
