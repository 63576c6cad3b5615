#!/usr/bin/env python
"""bench_filter.py — WHERE expressions on the GPU (ytgpu_evaluate_filter) and what the separate filter pass costs a GROUP BY.

  python bench_filter.py --steps K --warmup W [--rows N]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour.  N rows (10^8 by
default) of five columns:
  ts   int64 U[0, 10^9), a plain 64-bit vector
  d    double N(0, 1), a plain 64-bit vector
  k    int64 dictionary-encoded: 1-based uint32 indexes into 1000 values
  b    boolean as a bitmap (bit_width 1), p = 1/2
  url  URL-like strings of bench_groupby_strings.py: one of 64 prefixes, half of them "https://", then U[0, 48] letters
Filter legs (bitmap output only; kernel time from the library's CUDA events around the evaluation launch, median of the
steps; call time from CUDA events around the whole call):
  one_compare   ts >= a
  conjunction   ts >= a AND ts < b AND k IN (16 values) AND (d < x OR b)
  with_prefix   conjunction AND STARTS_WITH(url, "https://")
  contains      CONTAINS(url, "site4")                           (QL is_substr("site4", url))
  like          url LIKE 'https://www.site_.example.com/%q%'
Each leg reports its algorithmic bytes per row — the bytes of the column data it reads plus 1/8 byte of bitmap written
(the kernel evaluates every node for every row, so every referenced column is read) — and that traffic over the kernel
time, against the HBM peak.  A CONTAINS / LIKE leg reads the start (8) and length (4) of every row and the value bytes the
matcher consumes, which the bench counts exactly from the generated URLs: the matcher stops at a segment's earliest end
and an anchored segment stops at its first mismatch (MEASURED_PEAKS.json's when present, else the 3.35 TB/s data-sheet figure of the H100 SXM).
GROUP BY leg: two int64 keys (U[0, 1000) x U[0, 8)), SUM + MIN + MAX + AVG of an int64 column, through
ytgpu_scan_filter_groupby_multi with `ts >= a` as its built-in predicate against the filter pass + the bitmap as a
BOOLEAN column + the predicate {EQ, 1}; both results must be identical.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True  # the URL generator is imported from bench_groupby_strings.py: no __pycache__ in the tree
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py
DATASHEET_HBM_BPS = 3.35e12
AGG_SUM, AGG_MIN, AGG_MAX, AGG_AVG = 0, 1, 2, 4


def device_info():
    import torch
    power = None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        power = float(out.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return torch.cuda.get_device_properties(0).name, power


def hbm_peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        with open(path) as f:
            peaks = json.load(f)
        for key in ("hbm_bytes_per_s", "hbm_read_bytes_per_s", "dram_bytes_per_s"):
            if key in peaks:
                return float(peaks[key]), "MEASURED_PEAKS.json:" + key
    except Exception:
        pass
    return DATASHEET_HBM_BPS, "H100 SXM data sheet"


def _url_parts(heap, lengths):
    """The generated URLs are "https://www.site<k>.example.com/" (k < 64) + lowercase letters, in 96-byte slots."""
    import torch
    rows = heap.view(-1, 96)
    digit2 = (rows[:, 17] >= 48) & (rows[:, 17] <= 57)  # a two-digit site number
    site4 = rows[:, 16] == ord("4")
    one_digit = ~digit2
    tail = rows[:, 30:]
    valid = torch.arange(66, device=heap.device)[None, :] < (lengths.long() - 30)[:, None]
    isq = (tail == ord("q")) & valid
    has_q = isq.any(dim=1)
    first_q = torch.where(has_q, isq.to(torch.uint8).argmax(dim=1), lengths.long() - 31)  # index of the last byte when no q
    return site4, one_digit, has_q, first_q


def url_bytes_read(heap, lengths, chunk=1 << 24):
    """Mean value bytes the matcher consumes per row for CONTAINS(url, "site4") and the LIKE leg's pattern."""
    n = len(lengths)
    c_sum = l_sum = 0
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        site4, one_digit, _, first_q = _url_parts(heap[a * 96:b * 96], lengths[a:b])
        ln = lengths[a:b].long()
        c_sum += int((ln.where(~site4, 17)).sum().item())  # "site4" ends at byte 17; no letter tail holds a digit
        # the anchored first segment dies at byte 18 for a two-digit site; otherwise 30 bytes, then up to the first q
        l_sum += int(torch_where(one_digit, 30 + first_q + 1, 18).sum().item())
    return c_sum / n, l_sum / n


def url_counts(heap, lengths, chunk=1 << 24):
    """Rows the CONTAINS and LIKE legs select, from the generator's structure (a cross-check of the kernel's count)."""
    n = len(lengths)
    c = l_cnt = 0
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        site4, one_digit, has_q, _ = _url_parts(heap[a * 96:b * 96], lengths[a:b])
        c += int(site4.sum().item())
        l_cnt += int((one_digit & has_q).sum().item())
    return c, l_cnt


def torch_where(cond, a, b):
    import torch
    return torch.where(cond, a, torch.as_tensor(b, device=cond.device))


def median_ms(values):
    return round(statistics.median(values), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    import torch

    from bench_groupby_strings import url_strings
    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T
    assert torch.cuda.is_available(), "bench_filter.py needs a CUDA device"
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    ctx = GpuContext(0)
    n = args.rows
    name, power = device_info()
    peak, peak_src = hbm_peak()
    line = {"bench": "filter", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps, "warmup": args.warmup,
            "hbm_peak_bytes_per_s": peak, "hbm_peak_source": peak_src}

    ts = torch.randint(0, 10**9, (n,), device="cuda", generator=g)
    d = torch.randn(n, device="cuda", generator=g, dtype=torch.float64)
    kdict = torch.randint(-10**12, 10**12, (1000,), device="cuda", generator=g)
    kidx = torch.randint(1, 1001, (n,), device="cuda", generator=g, dtype=torch.int32)
    bbytes = torch.randint(0, 256, ((n + 63) // 64 * 8,), device="cuda", generator=g, dtype=torch.uint8)
    heap, starts, lengths = url_strings(n, g)
    cols = [Column(T.Int64, values=ts), Column(T.Double, values=d.view(torch.int64)),
            Column(T.Int64, values=kdict, dictionary_indexes=kidx, value_count=n),
            Column(T.Boolean, values=bbytes, bit_width=1, value_count=n)]
    strings = [(heap, starts, lengths, None)]
    TS, D, K, B, URL = 0, 1, 2, 3, 4
    lo, hi = 100_000_000, 900_000_000
    in_list = kdict[:16].cpu().numpy().view(np.uint64).tolist()
    x = np.float64(0.5).view(np.uint64).item()
    cmp_, in_, sw, and_, or_ = capi.FILTER_COMPARE, capi.FILTER_IN, capi.FILTER_STARTS_WITH, capi.FILTER_AND, capi.FILTER_OR
    one = [(cmp_, capi.CMP_GE, TS, 0, lo, 0)]
    conj = [(cmp_, capi.CMP_GE, TS, 0, lo, 0), (cmp_, capi.CMP_LT, TS, 0, hi, 0), (and_,), (in_, 0, K, 0, 0, 16), (and_,),
            (cmp_, capi.CMP_LT, D, 0, x, 0), (cmp_, capi.CMP_EQ, B, 0, 1, 0), (or_,), (and_,)]
    prefix = conj + [(sw, 0, URL, 0, 0, 8), (and_,)]
    consts = b"https://"
    needle, pattern = b"site4", b"https://www.site_.example.com/%q%"
    bitmap_write = 1 / 8
    read_contains, read_like = url_bytes_read(heap, lengths)
    legs = {
        "one_compare": (one, consts, 8 + bitmap_write),
        "conjunction": (conj, consts, 8 + 4 + 8 + 1 / 8 + bitmap_write),
        "with_prefix": (prefix, consts, 8 + 4 + 8 + 1 / 8 + 8 + 4 + 8 + bitmap_write),  # + starts, lengths, the 8 prefix bytes
        "contains": ([(capi.FILTER_CONTAINS, 0, URL, 0, 0, len(needle))], needle, 8 + 4 + read_contains + bitmap_write),
        "like": ([(capi.FILTER_LIKE, 0, URL, -1, 0, len(pattern))], pattern, 8 + 4 + read_like + bitmap_write),
    }
    line["url_mean_bytes"] = round(lengths.double().mean().item(), 4)
    ctx.enable_timers(True)
    for leg_name, (prog, leg_consts, bytes_per_row) in legs.items():
        def call(p=prog, c=leg_consts):
            return ctx.evaluate_filter(cols, strings, p, in_list, c, want_bytemap=False, want_rows=False)
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
        km = statistics.median(kernel)
        rate = n * bytes_per_row / (km * 1e-3)
        line[leg_name] = {"kernel_ms_median": median_ms(kernel), "kernel_ms_min": round(min(kernel), 4),
                          "call_ms_median": median_ms(calls), "selected": r["count"], "bytes_per_row": round(bytes_per_row, 4),
                          "bytes_per_s": rate, "share_of_hbm_peak": round(rate / peak, 4)}
    ctx.enable_timers(False)
    # parity of the one-comparison leg with torch
    line["one_compare"]["count_matches_torch"] = line["one_compare"]["selected"] == int((ts >= lo).sum().item())
    line["contains"]["count_matches_torch"], line["like"]["count_matches_torch"] = [
        line[k]["selected"] == c for k, c in zip(("contains", "like"), url_counts(heap, lengths))]
    del heap, starts, lengths, strings

    # GROUP BY: built-in predicate vs filter pass + bitmap column
    k0 = torch.randint(0, 1000, (n,), device="cuda", generator=g)
    k1 = torch.randint(0, 8, (n,), device="cuda", generator=g)
    v = torch.randint(-10**9, 10**9, (n,), device="cuda", generator=g)
    keys = [Column(T.Int64, values=k0), Column(T.Int64, values=k1)]
    aggs = [(AGG_SUM, 0), (AGG_MIN, 0), (AGG_MAX, 0), (AGG_AVG, 0)]
    vals = [Column(T.Int64, values=v), Column(T.Int64, values=ts)]

    def builtin():
        return ctx.scan_filter_groupby_multi(keys, vals, aggs, predicate=(capi.CMP_GE, lo), predicate_column=1, capacity=8000)

    def through_bitmap():
        f = ctx.evaluate_filter([cols[TS]], (), one, want_bytemap=False, want_rows=False)
        bm = Column(T.Boolean, values=f["bitmap"], bit_width=1, value_count=n)
        return ctx.scan_filter_groupby_multi(keys, [vals[0], bm], aggs, predicate=(capi.CMP_EQ, 1), predicate_column=1,
                                             capacity=8000)
    times = {"builtin_predicate": [], "filter_then_bitmap": []}
    for _ in range(args.warmup):
        builtin()
        through_bitmap()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.steps):  # alternate the two routes
        for key, fn in (("builtin_predicate", builtin), ("filter_then_bitmap", through_bitmap)):
            start.record()
            fn()
            stop.record()
            torch.cuda.synchronize()
            times[key].append(start.elapsed_time(stop))
    a, b = builtin(), through_bitmap()
    same = all(torch.equal(x, y) for x, y in zip(a["keys"] + a["values"] + a["value_null"] + [a["count"], a["first_row"]],
                                                 b["keys"] + b["values"] + b["value_null"] + [b["count"], b["first_row"]]))
    line["groupby_2keys_sum_min_max_avg"] = {"builtin_predicate_ms_median": median_ms(times["builtin_predicate"]),
                                             "filter_then_bitmap_ms_median": median_ms(times["filter_then_bitmap"]),
                                             "groups": len(a["count"]), "identical_results": same}
    ctx.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
