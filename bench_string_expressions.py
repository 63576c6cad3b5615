#!/usr/bin/env python
"""bench_string_expressions.py — computed string columns on the GPU (ytgpu_evaluate_expression_strings).

  python bench_string_expressions.py --steps K --warmup W [--rows N]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour.  N rows (10^8 by
default) of URL-like strings (bench_groupby_strings.url_strings: 30..84 bytes in 96-byte slots) whose letters are
upper-cased with probability 0.3, an int64 column a, and a host column of 1000 distinct mixed-case host names.
Legs (kernel time: the library's CUDA events around every launch of one call, median of the steps; a STRING result is one
call with a heap sized beforehand, so a size pass, a three-kernel scan and a fill pass):
  lower_url             lower(url)
  concat_url_x          concat(url, '/x')
  if_null_url           if_null(url, '') with 5 % of the rows NULL
  farm_hash_url         farm_hash(url)
  farm_hash_a_url_mod   farm_hash(a, url) % 64
  if_a_url_other        if(a > 0, url, 'other')          (a STRING IF: about half the rows keep url's piece)
  url_lt_site5          url < 'https://www.site5'        (a STRING COMPARE, BOOLEAN result)
  url_like              url like 'https://www.site_.example.com/%q%'   (LIKE over the url leaf: its one piece is matched as
                        contiguous bytes), beside filter_url_like: the same pattern as a ytgpu_evaluate_filter leaf
  lower_url_like_site4  lower(url) like '%site4%'        (fused: the matcher walks lower(url)'s piece under its case map),
                        beside lower_url_then_contains: lower(url) written out, then the filter's CONTAINS 'site4' over it
  if_substr_api         if(is_substr('/api/', url), 'api', 'web')   (a STRING result)
Algorithmic bytes per row: a string input reads its 8-byte start, 4-byte length and its bytes (+1 null byte when it has
NULLs), a numeric one 8 bytes; a STRING result writes its bytes, an 8-byte start, a 4-byte length and a null byte, a
numeric one 8 bytes and 1/8 byte of null bitmap; a COMPARE against a constant of c bytes reads at most c + 1 bytes of a
value; LIKE and CONTAINS are counted as reading every byte of the value, the most the matcher consumes.  That traffic over
the kernel time is set against the HBM peak
(MEASURED_PEAKS.json's when present, else the 3.35 TB/s data-sheet figure of the H100 SXM).
GROUP BY leg: COUNT and SUM of a grouped by lower(host), once computed (lower as one call into outputs allocated once, as
the string legs, then string_value_ids and the GROUP BY) and once over the host names lowered beforehand; both results must
be identical.  GpuContext.evaluate_expression is not used there: it runs a type and size query first, so a STRING result
would pay its size pass twice.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True  # helpers are imported from the other benchmarks: no __pycache__ in the tree
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_filter import SEED, device_info, hbm_peak, median_ms  # noqa: E402
from bench_groupby_strings import url_strings  # noqa: E402

AGG_SUM, AGG_COUNT = 0, 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    import numpy as np
    import torch

    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T
    from ytsaurus_b200.runtime import _string_column
    assert torch.cuda.is_available(), "bench_string_expressions.py needs a CUDA device"
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    ctx = GpuContext(0)
    n = args.rows
    name, power = device_info()
    peak, peak_src = hbm_peak()
    line = {"bench": "string_expressions", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps,
            "warmup": args.warmup, "hbm_peak_bytes_per_s": peak, "hbm_peak_source": peak_src}

    heap, starts, lengths = url_strings(n, g)
    chunk = 1 << 28
    for lo in range(0, heap.numel(), chunk):  # mixed case: 30 % of the letters upper-cased
        h = heap[lo:lo + chunk]
        up = (h >= 97) & (h <= 122) & (torch.rand(h.numel(), device="cuda", generator=g) < 0.3)
        h.sub_(up.to(torch.uint8) * 32)
    mean_len = float(lengths.double().mean())
    nulls = (torch.rand(n, device="cuda", generator=g) < 0.05).to(torch.uint8)
    a = torch.randint(-10**9, 10**9, (n,), device="cuda", generator=g)
    url = _string_column(heap, starts, lengths)
    url_nulls = _string_column(heap, starts, lengths, nulls)
    acol = Column(T.Int64, values=a)
    col, const, STR, U64, I64 = capi.EXPR_COLUMN, capi.EXPR_CONSTANT, int(T.String), int(T.Uint64), int(T.Int64)
    ec = capi.ExprConstants()
    ec.data += b"/xotherhttps://www.site5"  # "/x" at 0, "other" at 2, the URL bound at 7
    like_q, site4, api_needle = ec.string(b"https://www.site_.example.com/%q%"), ec.string(b"%site4%"), ec.string(b"/api/")
    api, web, site4_needle = ec.string(b"api"), ec.string(b"web"), ec.string(b"site4")
    consts = np.frombuffer(bytes(ec), np.uint8).copy()

    out_heap = torch.empty(int(heap.numel()) + 2 * n, dtype=torch.uint8, device="cuda")
    out_starts = torch.empty(n, dtype=torch.int64, device="cuda")
    out_lengths = torch.empty(n, dtype=torch.int32, device="cuda")
    out_nulls = torch.empty(n, dtype=torch.uint8, device="cuda")
    out_values = torch.empty(n, dtype=torch.int64, device="cuda")
    out_bitmap = torch.empty((n + 63) // 64 * 8, dtype=torch.uint8, device="cuda")

    def evaluate(prog, scols, numeric=()):
        """One ytgpu_evaluate_expression_strings call into the preallocated outputs -> (value type, heap bytes, NULL rows)."""
        sarr = (capi.StringColumn * len(scols))(*scols)
        views = [c.view() for c in numeric]
        carr = (capi.ColumnView * max(len(views), 1))(*views)
        nodes = (capi.ExprNode * len(prog))()
        for i, node in enumerate(prog):
            op, column, vtype, constant = (tuple(node) + (0,) * 4)[:4]
            nodes[i].op, nodes[i].column, nodes[i].type, nodes[i].constant = op, column, vtype, constant
        heap_bytes, vtype, nul = C.c_uint64(0), C.c_uint8(0), C.c_uint64(0)
        err = capi.Error()
        capi.check(ctx.lib.ytgpu_evaluate_expression_strings(
            ctx.handle, C.cast(carr, C.c_void_p), len(views), C.cast(sarr, C.c_void_p), len(scols), consts.ctypes.data, consts.size,
            C.cast(nodes, C.c_void_p), len(prog), None, out_values.data_ptr(), out_bitmap.data_ptr(), out_heap.data_ptr(),
            out_heap.numel(), out_starts.data_ptr(), out_lengths.data_ptr(), out_nulls.data_ptr(), C.byref(heap_bytes),
            C.byref(vtype), C.byref(nul), capi.MEM_DEVICE, C.byref(err)), err)
        return int(vtype.value), int(heap_bytes.value), int(nul.value)

    string_in, string_out, numeric_out = 12 + mean_len, mean_len + 13, 8 + 1 / 8
    legs = {
        "lower_url": ([(col, 0), (capi.EXPR_LOWER,)], [url], (), string_in + string_out),
        "concat_url_x": ([(col, 0), (const, 0, STR, 2), (capi.EXPR_CONCAT,)], [url], (), string_in + string_out + 2),
        "if_null_url": ([(col, 0), (const, 0, STR, 0), (capi.EXPR_IF_NULL, 0, STR)], [url_nulls], (),
                        (13 + 0.95 * mean_len) + (0.95 * mean_len + 13)),
        "farm_hash_url": ([(col, 0), (capi.EXPR_FARM_HASH, 1)], [url], (), string_in + numeric_out),
        "farm_hash_a_url_mod": ([(col, 0), (col, 1), (capi.EXPR_FARM_HASH, 2), (const, 0, U64, 64), (capi.EXPR_MOD,)], [url], [acol],
                                8 + string_in + numeric_out),
        "if_a_url_other": ([(col, 0), (const, 0, I64, 0), (capi.EXPR_COMPARE, capi.CMP_GT), (col, 1), (const, 0, STR, (2 << 32) | 5),
                            (capi.EXPR_IF,)], [url], [acol], 8 + 12 + 0.5 * mean_len + (0.5 * mean_len + 0.5 * 5 + 13)),
        "url_lt_site5": ([(col, 0), (const, 0, STR, (7 << 32) | 17), (capi.EXPR_COMPARE, capi.CMP_LT)], [url], (),
                         12 + 18 + numeric_out),
        "url_like": ([(col, 0), (capi.EXPR_LIKE, -1, 0, like_q)], [url], (), string_in + numeric_out),
        "lower_url_like_site4": ([(col, 0), (capi.EXPR_LOWER,), (capi.EXPR_LIKE, -1, 0, site4)], [url], (), string_in + numeric_out),
        "if_substr_api": ([(col, 0), (capi.EXPR_CONTAINS, 0, 0, api_needle), (const, 0, STR, api), (const, 0, STR, web), (capi.EXPR_IF,)],
                          [url], (), string_in + 3 + 13),
    }
    ctx.enable_timers(True)
    for leg_name, (prog, scols, numeric, bytes_per_row) in legs.items():
        for _ in range(args.warmup):
            evaluate(prog, scols, numeric)
        kernel, calls = [], []
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.steps):
            ctx.reset_timers()
            start.record()
            vtype, size, nul = evaluate(prog, scols, numeric)
            stop.record()
            torch.cuda.synchronize()
            kernel.append(ctx.kernel_ms(capi.KC_DECODE)[0] + ctx.kernel_ms(capi.KC_GATHER)[0])
            calls.append(start.elapsed_time(stop))
        km = statistics.median(kernel)
        rate = n * bytes_per_row / (km * 1e-3)
        line[leg_name] = {"kernel_ms_median": median_ms(kernel), "kernel_ms_min": round(min(kernel), 4), "call_ms_median": median_ms(calls),
                          "result_type": vtype, "heap_bytes": size, "null_count": nul, "bytes_per_row": round(bytes_per_row, 4),
                          "bytes_per_s": rate, "share_of_hbm_peak": round(rate / peak, 4)}
    # the filter's LIKE over the same column, and lower(url) written out then the filter's CONTAINS: the routes the fused
    # legs replace
    def filter_bitmap(scol, op, constant, escape=-1):
        return ctx.evaluate_filter([], [scol], [(op, 0, 0, escape, constant >> 32, constant & 0xFFFFFFFF)], string_constants=bytes(ec),
                                   want_bytemap=False, want_rows=False)["bitmap"]
    routes = {
        "filter_url_like": (lambda: filter_bitmap((heap, starts, lengths, None), capi.FILTER_LIKE, like_q), string_in + 1 / 8),
        "lower_url_then_contains": (lambda: (evaluate(legs["lower_url"][0], [url]),
                                             filter_bitmap((out_heap, out_starts, out_lengths, None), capi.FILTER_CONTAINS, site4_needle))[1],
                                    (string_in + string_out) + (12 + mean_len + 1 / 8)),
    }
    bitmaps = {}
    for leg_name, (fn, bytes_per_row) in routes.items():
        for _ in range(args.warmup):
            fn()
        kernel, calls = [], []
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.steps):
            ctx.reset_timers()
            start.record()
            bitmaps[leg_name] = fn()
            stop.record()
            torch.cuda.synchronize()
            kernel.append(ctx.kernel_ms(capi.KC_DECODE)[0] + ctx.kernel_ms(capi.KC_GATHER)[0])
            calls.append(start.elapsed_time(stop))
        km = statistics.median(kernel)
        rate = n * bytes_per_row / (km * 1e-3)
        line[leg_name] = {"kernel_ms_median": median_ms(kernel), "kernel_ms_min": round(min(kernel), 4), "call_ms_median": median_ms(calls),
                          "bytes_per_row": round(bytes_per_row, 4), "bytes_per_s": rate, "share_of_hbm_peak": round(rate / peak, 4)}
    ctx.enable_timers(False)
    # the fused legs select the rows of the routes they replace (no NULLs here: TRUE rows are the value bits)
    for leg_name, route in (("url_like", "filter_url_like"), ("lower_url_like_site4", "lower_url_then_contains")):
        evaluate(legs[leg_name][0], [url])
        word = torch.arange(64, device="cuda", dtype=torch.int64)
        vals = torch.zeros((n + 63) // 64 * 64, dtype=torch.int64, device="cuda")
        vals[:n] = out_values
        packed = (vals.view(-1, 64) << word).sum(1)
        line[leg_name]["matches_" + route] = bool(torch.equal(packed, bitmaps[route].view(torch.int64)))
    # lower(url) against torch's ASCII lowering of the same slots
    evaluate(legs["lower_url"][0], [url])
    ref = heap.view(n, -1)[:1_000_000].clone()
    ref += ((ref >= 65) & (ref <= 90)).to(torch.uint8) * 32
    rows = torch.arange(1_000_000, device="cuda")
    got_ok = bool(torch.equal(out_lengths[:1_000_000], lengths[:1_000_000]))
    pos = out_starts[:1_000_000]
    for j in range(0, 30):  # the first 30 bytes of every value (each is at least 30 long)
        got_ok &= bool(torch.equal(out_heap[pos + j], ref[rows, j]))
    line["lower_url"]["matches_torch_first_10e6_rows"] = got_ok
    del ref

    # GROUP BY lower(host): 1000 mixed-case host names, computed against precomputed
    names = [b"Host-%03d.Example.%s" % (k, [b"COM", b"org", b"Net"][k % 3]) for k in range(1000)]
    table = np.frombuffer(b"".join(names), np.uint8)
    offs = np.cumsum([0] + [len(x) for x in names[:-1]]).astype(np.int64)
    pick = torch.randint(0, 1000, (n,), device="cuda", generator=g)
    hstarts = torch.from_numpy(offs).cuda()[pick]
    hlens = torch.tensor([len(x) for x in names], dtype=torch.int32, device="cuda")[pick]
    hheap = torch.from_numpy(table.copy()).cuda()
    lheap = torch.from_numpy(np.frombuffer(b"".join(x.lower() for x in names), np.uint8).copy()).cuda()
    aggs = [(AGG_COUNT, 0), (AGG_SUM, 0)]
    vcols = [acol]

    hcol = _string_column(hheap, hstarts, hlens)

    def computed():
        evaluate([(col, 0), (capi.EXPR_LOWER,)], [hcol])
        ids, _ = ctx.string_value_ids(out_heap, out_starts, out_lengths, out_nulls)
        return ctx.scan_filter_groupby_multi([Column(U64, values=ids, value_count=n)], vcols, aggs, capacity=4096)

    def precomputed():
        ids, _ = ctx.string_value_ids(lheap, hstarts, hlens)
        return ctx.scan_filter_groupby_multi([Column(U64, values=ids, value_count=n)], vcols, aggs, capacity=4096)
    times = {"computed_key": [], "precomputed_key": []}
    for _ in range(args.warmup):
        computed()
        precomputed()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.steps):  # alternate the two routes
        for key, fn in (("computed_key", computed), ("precomputed_key", precomputed)):
            start.record()
            fn()
            stop.record()
            torch.cuda.synchronize()
            times[key].append(start.elapsed_time(stop))
    x, y = computed(), precomputed()
    same = all(torch.equal(p, q) for p, q in zip(x["keys"] + x["key_null"] + x["values"] + x["value_null"] + [x["count"], x["first_row"]],
                                                 y["keys"] + y["key_null"] + y["values"] + y["value_null"] + [y["count"], y["first_row"]]))
    line["groupby_lower_host_count_sum"] = {"computed_key_ms_median": median_ms(times["computed_key"]),
                                            "precomputed_key_ms_median": median_ms(times["precomputed_key"]),
                                            "groups": len(x["count"]), "identical_results": same}
    ctx.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
