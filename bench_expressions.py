#!/usr/bin/env python
"""bench_expressions.py — computed columns on the GPU (ytgpu_evaluate_expression) and what the separate pass costs a GROUP BY.

  python bench_expressions.py --steps K --warmup W [--rows N]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour.  N rows (10^8 by
default) of plain 64-bit columns: a, b int64 U[-10^9, 10^9); price double U[0, 100); qty double U[0, 10); d double N(0, 1).
Expression legs (kernel time from the library's CUDA events around the evaluation launch, median of the steps; call time
from CUDA events around the whole call):
  add           a + b
  mod_1000      a % 1000                       (64-bit integer division is a software sequence on the GPU)
  mul_double    price * qty
  cast_div      int64(d * 100.0) / 7
  chain_16      a 16-node chain over a and b: ((((a + b) * 3 - a) ^ 5) + b) & c | a, negated
  guarded_div   if(b = 0, 0, a / b)            (a division whose zero divisors the IF guards; b has zeros here)
  if_bucket     if(a < 0, 0, if(a < 5 * 10^8, 1, 2))   (a two-level if)
  and_signs     (a > 0) AND (b < 0)            (a BOOLEAN result)
  in_16         if(k in (16 int64 entries), b, 0)   with k int64 U[0, 64): a quarter of the rows match (the numeric-IN
                kernel: a binary search over the list staged in shared memory)
Each leg reports its algorithmic bytes per row — 8 per referenced column read, plus 8 bytes of value and 1/8 byte of null
bitmap written — and that traffic over the kernel time, against the HBM peak (MEASURED_PEAKS.json's when present, else
the 3.35 TB/s data-sheet figure of the H100 SXM).
GROUP BY leg: keys (a % 1000, k) with k int64 U[0, 8), SUM + MIN of b, once through the computed column and once with the
same key precomputed by torch.fmod (C's %); both results must be identical.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True  # helpers are imported from bench_filter.py: no __pycache__ in the tree
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_filter import SEED, device_info, hbm_peak, median_ms  # noqa: E402

AGG_SUM, AGG_MIN = 0, 1


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
    assert torch.cuda.is_available(), "bench_expressions.py needs a CUDA device"
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    ctx = GpuContext(0)
    n = args.rows
    name, power = device_info()
    peak, peak_src = hbm_peak()
    line = {"bench": "expressions", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps, "warmup": args.warmup,
            "hbm_peak_bytes_per_s": peak, "hbm_peak_source": peak_src}

    a = torch.randint(-10**9, 10**9, (n,), device="cuda", generator=g)
    b = torch.randint(-10**9, 10**9, (n,), device="cuda", generator=g)
    bz = torch.where(b % 16 == 0, torch.zeros_like(b), b)  # b with zero divisors in 1/16 of the rows
    price = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * 100
    qty = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * 10
    d = torch.randn(n, device="cuda", generator=g, dtype=torch.float64)
    k = torch.randint(0, 64, (n,), device="cuda", generator=g)
    cols = [Column(T.Int64, values=a), Column(T.Int64, values=b), Column(T.Double, values=price.view(torch.int64)),
            Column(T.Double, values=qty.view(torch.int64)), Column(T.Double, values=d.view(torch.int64)), Column(T.Int64, values=bz),
            Column(T.Int64, values=k)]
    A, B, PRICE, QTY, D, BZ, K = range(7)
    in_consts = capi.ExprConstants()
    in_list = in_consts.in_list(range(0, 64, 4))
    col, const, cast = capi.EXPR_COLUMN, capi.EXPR_CONSTANT, capi.EXPR_CAST
    cmp, iff = capi.EXPR_COMPARE, capi.EXPR_IF
    i64, f64 = int(T.Int64), int(T.Double)

    def dbl(x):
        return int(np.float64(x).view(np.uint64))
    chain = [(col, A), (col, B), (capi.EXPR_ADD,), (const, 0, i64, 3), (capi.EXPR_MUL,), (col, A), (capi.EXPR_SUB,),
             (const, 0, i64, 5), (capi.EXPR_BIT_XOR,), (col, B), (capi.EXPR_ADD,), (const, 0, i64, 0x7FFFFFFF), (capi.EXPR_BIT_AND,),
             (col, A), (capi.EXPR_BIT_OR,), (capi.EXPR_NEG,)]
    assert len(chain) == 16
    written = 8 + 1 / 8
    legs = {
        "add": ([(col, A), (col, B), (capi.EXPR_ADD,)], 16 + written),
        "mod_1000": ([(col, A), (const, 0, i64, 1000), (capi.EXPR_MOD,)], 8 + written),
        "mul_double": ([(col, PRICE), (col, QTY), (capi.EXPR_MUL,)], 16 + written),
        "cast_div": ([(col, D), (const, 0, f64, dbl(100.0)), (capi.EXPR_MUL,), (cast, 0, i64), (const, 0, i64, 7), (capi.EXPR_DIV,)],
                     8 + written),
        "chain_16": (chain, 16 + written),
        "guarded_div": ([(col, BZ), (const, 0, i64, 0), (cmp, capi.CMP_EQ), (const, 0, i64, 0), (col, A), (col, BZ), (capi.EXPR_DIV,),
                         (iff,)], 16 + written),
        "if_bucket": ([(col, A), (const, 0, i64, 0), (cmp, capi.CMP_LT), (const, 0, i64, 0), (col, A), (const, 0, i64, 5 * 10**8),
                       (cmp, capi.CMP_LT), (const, 0, i64, 1), (const, 0, i64, 2), (iff,), (iff,)], 8 + written),
        "and_signs": ([(col, A), (const, 0, i64, 0), (cmp, capi.CMP_GT), (col, B), (const, 0, i64, 0), (cmp, capi.CMP_LT), (capi.EXPR_AND,)],
                      16 + written),
        "in_16": ([(col, K), (capi.EXPR_IN, 0, 0, in_list), (col, B), (const, 0, i64, 0), (iff,)], 16 + written, bytes(in_consts)),
    }
    ctx.enable_timers(True)
    results = {}
    for leg_name, (prog, bytes_per_row, *consts) in legs.items():
        def call(p=prog, c=consts[0] if consts else b""):
            return ctx.evaluate_expression(cols, p, string_constants=c)
        for _ in range(args.warmup):
            call()
        kernel, calls = [], []
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.steps):
            ctx.reset_timers()
            start.record()
            r = call()
            stop.record()
            torch.cuda.synchronize()
            kernel.append(ctx.kernel_ms(capi.KC_DECODE)[0])
            calls.append(start.elapsed_time(stop))
        results[leg_name] = r
        km = statistics.median(kernel)
        rate = n * bytes_per_row / (km * 1e-3)
        line[leg_name] = {"kernel_ms_median": median_ms(kernel), "kernel_ms_min": round(min(kernel), 4),
                          "call_ms_median": median_ms(calls), "null_count": r["null_count"], "bytes_per_row": round(bytes_per_row, 4),
                          "bytes_per_s": rate, "share_of_hbm_peak": round(rate / peak, 4)}
    ctx.enable_timers(False)
    # parity of two legs with torch
    line["add"]["matches_torch"] = bool(torch.equal(results["add"]["values"], a + b))
    line["mod_1000"]["matches_torch"] = bool(torch.equal(results["mod_1000"]["values"], torch.fmod(a, 1000)))
    line["in_16"]["matches_torch"] = bool(torch.equal(results["in_16"]["values"], torch.where(k % 4 == 0, b, torch.zeros_like(b))))
    safe = torch.where(bz == 0, torch.ones_like(bz), bz)
    line["guarded_div"]["matches_torch"] = bool(torch.equal(results["guarded_div"]["values"],
                                                            torch.where(bz == 0, torch.zeros_like(a), torch.div(a, safe, rounding_mode="trunc"))))
    line["if_bucket"]["matches_torch"] = bool(torch.equal(results["if_bucket"]["values"],
                                                          torch.where(a < 0, 0, torch.where(a < 5 * 10**8, 1, 2))))
    line["and_signs"]["matches_torch"] = bool(torch.equal(results["and_signs"]["values"], ((a > 0) & (b < 0)).to(torch.int64)))
    del results, price, qty, d, bz, safe

    # GROUP BY over (a % 1000, k): the computed key against the same key precomputed
    k = torch.randint(0, 8, (n,), device="cuda", generator=g)
    kcol, vcols = Column(T.Int64, values=k), [Column(T.Int64, values=b)]
    aggs = [(AGG_SUM, 0), (AGG_MIN, 0)]
    mod_prog = legs["mod_1000"][0]
    pre = Column(T.Int64, values=torch.fmod(a, 1000))

    def computed():
        key = ctx.evaluate_expression(cols[:1], mod_prog)["column"]
        return ctx.scan_filter_groupby_multi([key, kcol], vcols, aggs, capacity=20000)

    def precomputed():
        return ctx.scan_filter_groupby_multi([pre, kcol], vcols, aggs, capacity=20000)
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
    line["groupby_mod1000_and_k_sum_min"] = {"computed_key_ms_median": median_ms(times["computed_key"]),
                                             "precomputed_key_ms_median": median_ms(times["precomputed_key"]),
                                             "groups": len(x["count"]), "identical_results": same}
    ctx.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
