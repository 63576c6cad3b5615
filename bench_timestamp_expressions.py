#!/usr/bin/env python
"""bench_timestamp_expressions.py — timestamp_floor_* and format_timestamp as computed columns on the GPU.

  python bench_timestamp_expressions.py --steps K --warmup W [--rows N]

N rows (10^8 by default) of int64 timestamps uniform over 2015-01-01 .. 2025-01-01, generated on the device from a fixed
seed and passed in the DEVICE memory flavour.  Legs (kernel time: the library's CUDA events around every launch of one
call, median of the steps; a STRING result is one call with a heap sized beforehand: a size pass, a three-kernel scan and a
fill pass):
  floor_hour .. floor_year   timestamp_floor_<unit>(ts)                   (ytgpu_evaluate_expression)
  format_date                format_timestamp(ts, '%Y-%m-%d')
  format_datetime            format_timestamp(ts, '%Y-%m-%dT%H:%M:%S')
  format_month_eq            format_timestamp(ts, '%Y-%m') = '2024-03'    (a BOOLEAN result)
Algorithmic bytes per row: 8 read; a numeric result writes 8 bytes and 1/8 byte of null bitmap; a STRING result its bytes,
an 8-byte start, a 4-byte length and a null byte.  That traffic over the kernel time is set against the HBM peak
(MEASURED_PEAKS.json's when present, else the 3.35 TB/s data-sheet figure of the H100 SXM).
Each leg checks its result on 10^6 sampled rows: the floors against numpy (datetime64[M] / [Y] casts for the month and
year, integer arithmetic for the hour, day and the Monday week), the formats byte for byte against time.strftime over
time.gmtime.
GROUP BY leg: COUNT and SUM of an int64 b grouped by timestamp_floor_day(ts), end to end (the floor into a column
allocated once, then scan_filter_groupby_multi), alternated with the same GROUP BY over day keys computed beforehand;
both results must be identical.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True  # helpers are imported from the other benchmarks: no __pycache__ in the tree
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_filter import SEED, device_info, hbm_peak, median_ms  # noqa: E402

AGG_SUM, AGG_COUNT = 0, 3

T0, T1 = 1420070400, 1735689600  # 2015-01-01, 2025-01-01


def floor_numpy(unit, t):
    import numpy as np
    if unit == 0:
        return t - t % 3600
    d = t // 86400
    if unit == 1:
        return d * 86400
    if unit == 2:
        return (d - (d + 3) % 7) * 86400
    cast = "datetime64[M]" if unit == 3 else "datetime64[Y]"
    return t.astype("datetime64[s]").astype(cast).astype("datetime64[s]").astype(np.int64)


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
    assert torch.cuda.is_available(), "bench_timestamp_expressions.py needs a CUDA device"
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    ctx = GpuContext(0)
    n = args.rows
    name, power = device_info()
    peak, peak_src = hbm_peak()
    line = {"bench": "timestamp_expressions", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps,
            "warmup": args.warmup, "hbm_peak_bytes_per_s": peak, "hbm_peak_source": peak_src}
    ts = torch.randint(T0, T1, (n,), device="cuda", generator=g)
    tcol = Column(T.Int64, values=ts)
    sample = torch.randint(0, n, (1_000_000,), device="cuda", generator=g)
    ts_sample = ts[sample].cpu().numpy()
    col, const, STR = capi.EXPR_COLUMN, capi.EXPR_CONSTANT, int(T.String)
    ec = capi.ExprConstants()
    f_date, f_datetime, f_month, march = ec.string(b"%Y-%m-%d"), ec.string(b"%Y-%m-%dT%H:%M:%S"), ec.string(b"%Y-%m"), ec.string(b"2024-03")
    consts = np.frombuffer(bytes(ec), np.uint8).copy()

    out_heap = torch.empty(20 * n, dtype=torch.uint8, device="cuda")
    out_starts = torch.empty(n, dtype=torch.int64, device="cuda")
    out_lengths = torch.empty(n, dtype=torch.int32, device="cuda")
    out_nulls = torch.empty(n, dtype=torch.uint8, device="cuda")
    out_values = torch.empty(n, dtype=torch.int64, device="cuda")
    out_bitmap = torch.empty((n + 63) // 64 * 8, dtype=torch.uint8, device="cuda")
    carr = (capi.ColumnView * 1)(tcol.view())

    def evaluate(prog, strings):
        nodes = (capi.ExprNode * len(prog))()
        for i, node in enumerate(prog):
            op, column, vtype, constant = (tuple(node) + (0,) * 4)[:4]
            nodes[i].op, nodes[i].column, nodes[i].type, nodes[i].constant = op, column, vtype, constant
        heap_bytes, vtype, nul = C.c_uint64(0), C.c_uint8(0), C.c_uint64(0)
        err = capi.Error()
        if not strings:
            capi.check(ctx.lib.ytgpu_evaluate_expression(ctx.handle, C.cast(carr, C.c_void_p), 1, C.cast(nodes, C.c_void_p), len(prog), None,
                                                         out_values.data_ptr(), out_bitmap.data_ptr(), C.byref(vtype), C.byref(nul),
                                                         capi.MEM_DEVICE, C.byref(err)), err)
            return int(vtype.value), 0, int(nul.value)
        capi.check(ctx.lib.ytgpu_evaluate_expression_strings(
            ctx.handle, C.cast(carr, C.c_void_p), 1, None, 0, consts.ctypes.data, consts.size, C.cast(nodes, C.c_void_p), len(prog), None,
            out_values.data_ptr(), out_bitmap.data_ptr(), out_heap.data_ptr(), out_heap.numel(), out_starts.data_ptr(),
            out_lengths.data_ptr(), out_nulls.data_ptr(), C.byref(heap_bytes), C.byref(vtype), C.byref(nul), capi.MEM_DEVICE,
            C.byref(err)), err)
        return int(vtype.value), int(heap_bytes.value), int(nul.value)

    def check_floor(unit):
        got = out_values[sample].cpu().numpy()
        assert np.array_equal(got, floor_numpy(unit, ts_sample)), unit

    def check_format(fmt):  # every value of these formats has one length over years 1000 .. 9999
        want = [time.strftime(fmt, time.gmtime(int(x))).encode() for x in ts_sample]
        width = len(want[0])
        assert bool((out_lengths[sample] == width).all()), fmt
        pos = out_starts[sample].unsqueeze(1) + torch.arange(width, device="cuda")
        got = out_heap[pos].cpu().numpy()
        assert np.array_equal(got, np.frombuffer(b"".join(want), np.uint8).reshape(-1, width)), fmt

    def check_march():
        got = out_values[sample].cpu().numpy()
        want = (ts_sample >= 1709251200) & (ts_sample < 1711929600)
        assert np.array_equal(got, want.astype(np.int64))

    numeric_out, string_out = 8 + 1 / 8, 13
    legs = {}
    for unit, leg in enumerate(["floor_hour", "floor_day", "floor_week", "floor_month", "floor_year"]):
        legs[leg] = ([(col, 0), (capi.EXPR_TIMESTAMP_FLOOR, unit)], False, 8 + numeric_out, lambda u=unit: check_floor(u))
    legs["format_date"] = ([(col, 0), (capi.EXPR_FORMAT_TIMESTAMP, 0, 0, f_date)], True, 8 + 10 + string_out,
                           lambda: check_format("%Y-%m-%d"))
    legs["format_datetime"] = ([(col, 0), (capi.EXPR_FORMAT_TIMESTAMP, 0, 0, f_datetime)], True, 8 + 19 + string_out,
                               lambda: check_format("%Y-%m-%dT%H:%M:%S"))
    legs["format_month_eq"] = ([(col, 0), (capi.EXPR_FORMAT_TIMESTAMP, 0, 0, f_month), (const, 0, STR, march),
                                (capi.EXPR_COMPARE, capi.CMP_EQ)], True, 8 + numeric_out, check_march)
    ctx.enable_timers(True)
    for leg_name, (prog, strings, bytes_per_row, check) in legs.items():
        for _ in range(args.warmup):
            evaluate(prog, strings)
        kernel, calls = [], []
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.steps):
            ctx.reset_timers()
            start.record()
            vtype, size, nul = evaluate(prog, strings)
            stop.record()
            torch.cuda.synchronize()
            kernel.append(ctx.kernel_ms(capi.KC_DECODE)[0] + ctx.kernel_ms(capi.KC_GATHER)[0])
            calls.append(start.elapsed_time(stop))
        check()
        km = statistics.median(kernel)
        rate = n * bytes_per_row / (km * 1e-3)
        line[leg_name] = {"kernel_ms_median": median_ms(kernel), "kernel_ms_min": round(min(kernel), 4), "call_ms_median": median_ms(calls),
                          "result_type": vtype, "heap_bytes": size, "null_count": nul, "bytes_per_row": round(bytes_per_row, 4),
                          "bytes_per_s": rate, "share_of_hbm_peak": round(rate / peak, 4), "checked": True}
    ctx.enable_timers(False)

    # GROUP BY timestamp_floor_day(ts) with COUNT and SUM(b), end to end: the floor into a column, then the GROUP BY over
    # it; beside the same GROUP BY over day keys computed beforehand with torch.  Both results must be identical.
    b = Column(T.Int64, values=torch.randint(0, 1000, (n,), device="cuda", generator=g))
    aggs = [(AGG_COUNT, 0), (AGG_SUM, 0)]
    days = ts - ts % 86400

    def computed():
        evaluate([(col, 0), (capi.EXPR_TIMESTAMP_FLOOR, capi.TIMESTAMP_DAY)], False)
        return ctx.scan_filter_groupby_multi([Column(T.Int64, values=out_values, value_count=n)], [b], aggs, capacity=8192)

    def precomputed():
        return ctx.scan_filter_groupby_multi([Column(T.Int64, values=days, value_count=n)], [b], aggs, capacity=8192)
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
    assert same, "GROUP BY timestamp_floor_day(ts) differs from the GROUP BY over precomputed days"
    line["groupby_floor_day_count_sum"] = {"computed_key_ms_median": median_ms(times["computed_key"]),
                                           "precomputed_key_ms_median": median_ms(times["precomputed_key"]),
                                           "groups": len(x["count"]), "identical_results": same}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
