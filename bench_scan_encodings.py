"""TPC-H Q1 through NativeScan over one lineitem written in different Parquet value encodings.

Writes the lineitem the way bench.py's e2e leg does -- in-memory file images in pinned host memory, 1 Mi-row row groups, INT64
decimals -- once per layout:
  dictionary  every column dictionary-encoded (the writers' default; bench.py's e2e default)
  plain       PLAIN numerics, dictionary flags
  delta       DELTA_BINARY_PACKED money / date columns, dictionary flags (parquet-mr's v2 writer)
  bss         f64 money as BYTE_STREAM_SPLIT, dictionary flags; compared with plain_f64 (PLAIN f64 money)
and reports per layout: file bytes, H2D bytes and ms per step, rows/s, the copy-stream and decode-stream time per batch (from the
scan's CB200_TRACE lines, in a child process so that tracing does not touch the timed steps), and -- in a torch.profiler run -- the
time of the decode kernels with their algorithmic bandwidth (encoded bytes in + decoded bytes out) against the H100's 3.35 TB/s.
Prints one JSON line.  Q1 outputs must agree bit for bit across dictionary / plain / delta, and between bss and plain_f64."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "datafusion-comet_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np

LAYOUTS = ["dictionary", "plain", "delta", "bss", "plain_f64"]
MONEY = ["l_quantity", "l_extendedprice", "l_discount", "l_tax"]
HBM_TBPS = 3.35


def layout_images(args, layout):
    """-> list of Parquet images (bytes) of the lineitem in `layout`"""
    import pyarrow as pa
    import pyarrow.parquet as pq
    from comet_b200 import tpch
    variant = "f64" if layout in ("bss", "plain_f64") else "dec"
    cols = tpch.gen_lineitem(args.rows, seed=args.seed)
    tbl = tpch.lineitem_table(cols, variant, dictionary=True)
    flags = ["l_returnflag", "l_linestatus"]
    kw = {"use_dictionary": True} if layout == "dictionary" else {"use_dictionary": flags}
    if layout == "delta":
        kw["column_encoding"] = {k: "DELTA_BINARY_PACKED" for k in MONEY + ["l_shipdate"]}
    elif layout == "bss":
        kw["column_encoding"] = {k: "BYTE_STREAM_SPLIT" for k in MONEY}
    per = (args.rows + args.files - 1) // args.files
    out = []
    for i in range(args.files):
        sink = pa.BufferOutputStream()
        pq.write_table(tbl.slice(i * per, per), sink, row_group_size=1 << 20, compression="NONE", data_page_version="1.0",
                       store_decimal_as_integer=True, **kw)
        out.append(sink.getvalue().to_pybytes())
    return variant, out


def register(native, torch, layout, images):
    pinned, files = [], []
    for i, b in enumerate(images):
        h = torch.empty(len(b), dtype=torch.uint8, pin_memory=True)
        h.numpy()[:] = np.frombuffer(b, dtype=np.uint8)
        pinned.append(h)
        files.append(native.register_memory_file(f"enc-{layout}-{i}", h))
    return pinned, files


def q1_step(native, tpch, variant, files, chunk_rows):
    with native.Plan(tpch.q1_partial_plan(variant, scan=tpch.q1_native_scan(variant, files)), [], config={"spark.comet.b200.chunkRows": str(chunk_rows)}) as p:
        state = p.collect()
        st = p.stats()
    with native.Plan(tpch.q1_final_plan(variant), [state]) as p:
        res = p.collect()
    return res, st


def canonical(res):
    rows = sorted(res.to_pylist(), key=lambda r: (r["col_0"], r["col_1"]))
    return json.dumps(rows, default=lambda x: repr(x) if not isinstance(x, float) else float(x).hex())


def trace_child(args):
    """one warm step and one traced step of one layout; prints the mean copy / decode stream time per batch as JSON"""
    import torch
    from comet_b200 import native, tpch
    variant, images = layout_images(args, args.trace_layout)
    _, files = register(native, torch, args.trace_layout, images)
    q1_step(native, tpch, variant, files, args.chunk_rows)
    print(json.dumps({"ready": True}), flush=True)
    q1_step(native, tpch, variant, files, args.chunk_rows)


def measure_trace(args, layout):
    env = dict(os.environ, CB200_TRACE="1")
    cmd = [sys.executable, os.path.abspath(__file__), "--trace-layout", layout, "--rows", str(args.rows), "--files", str(args.files),
           "--seed", str(args.seed), "--chunk-rows", str(args.chunk_rows)]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=tempfile.gettempdir())
    if p.returncode != 0:
        return {"error": p.stderr[-500:]}
    err = p.stderr
    err = err[err.rfind("parquet scan:"):]                  # the traced (second) step only
    pat = re.compile(r"batch of (\d+) rows: copy stream ([\d.]+) ms, decode stream \(waits \+ decode\) ([\d.]+) ms")
    b = [(int(r), float(c), float(d)) for r, c, d in pat.findall(err)]
    if not b:
        return {"error": "no trace lines"}
    full = [x for x in b if x[0] == max(y[0] for y in b)]
    return {"batches": len(b), "rows_per_batch": full[0][0], "copy_ms_per_batch": sum(x[1] for x in full) / len(full),
            "decode_ms_per_batch": sum(x[2] for x in full) / len(full)}


def profile_kernels(torch, native, tpch, variant, files, chunk_rows):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        q1_step(native, tpch, variant, files, chunk_rows)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "k_pq_" in e.key:
            name = re.sub(r"^void |cb200::|\(.*$", "", e.key)
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            out[name] = {"ms": t / 1e3, "calls": e.count}
    return out


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 25)
    ap.add_argument("--files", type=int, default=16)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--chunk-rows", type=int, default=1 << 23)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--layouts", default=",".join(LAYOUTS))
    ap.add_argument("--trace-layout", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.trace_layout:
        return trace_child(args)
    import torch
    from comet_b200 import native, tpch
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": args.rows, "files": args.files, "chunk_rows": args.chunk_rows,
           "layouts": {}}
    outputs = {}
    for layout in args.layouts.split(","):
        variant, images = layout_images(args, layout)
        pinned, files = register(native, torch, layout, images)
        file_bytes = sum(len(b) for b in images)
        del images
        for _ in range(args.warmup):
            q1_step(native, tpch, variant, files, args.chunk_rows)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        h2d = 0
        for _ in range(args.steps):
            out, st = q1_step(native, tpch, variant, files, args.chunk_rows)
            h2d += st["h2d_bytes"]
        el = time.perf_counter() - t0
        outputs[layout] = canonical(out)
        r = {"file_bytes": file_bytes, "h2d_bytes_per_step": h2d // args.steps, "ms_per_step": 1e3 * el / args.steps, "rows_per_s": args.rows * args.steps / el}
        r["kernels"] = profile_kernels(torch, native, tpch, variant, files, args.chunk_rows)
        enc_cols = {"delta": MONEY + ["l_shipdate"], "bss": MONEY}.get(layout)
        if enc_cols:  # algorithmic bytes of the new decoders: the encoded column chunks in + the decoded values out
            import pyarrow as pa
            import pyarrow.parquet as pq
            enc_in = 0
            for h in pinned:
                md = pq.ParquetFile(pa.BufferReader(h.numpy().tobytes())).metadata
                for g in range(md.num_row_groups):
                    for c in range(md.num_columns):
                        if md.schema.column(c).name in enc_cols:
                            enc_in += md.row_group(g).column(c).total_compressed_size
            dec_out = args.rows * sum(4 if k == "l_shipdate" else 8 for k in enc_cols)
            names = [k for k in r["kernels"] if ("dbp" in k if layout == "delta" else "k_pq_plain" in k)]
            ms = sum(r["kernels"][k]["ms"] for k in names)
            r["decoder"] = {"kernels": names, "ms_per_step": ms, "bytes": enc_in + dec_out,
                            "TBps": (enc_in + dec_out) / (ms * 1e-3) / 1e12 if ms > 0 else None}
            r["decoder"]["of_hbm_peak"] = r["decoder"]["TBps"] / HBM_TBPS if r["decoder"]["TBps"] else None
        for f in files:
            native.register_memory_file(f[len("memory://"):], None)
        del pinned
        r["trace"] = measure_trace(args, layout)
        res["layouts"][layout] = r
    same = [k for k in ("dictionary", "plain", "delta") if k in outputs]
    res["outputs_identical_dec"] = len({outputs[k] for k in same}) <= 1
    if "bss" in outputs and "plain_f64" in outputs:
        res["outputs_identical_f64"] = outputs["bss"] == outputs["plain_f64"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
