#!/usr/bin/env python
"""bench_groupby_strings.py — GROUP BY with string-valued aggregates (ytgpu_scan_filter_groupby_multi_strings).

  python bench_groupby_strings.py --steps K --warmup W [--rows N] [--scalar-only]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour.
String legs, N rows (10^8 by default):
  URL-like strings: one of 64 prefixes "https://www.site<k>.example.com/" + a tail of U[0, 48] lower-case letters, each in
  a 96-byte slot of the heap.  One int64 key column with U[0, G) for G = 10^3 and 10^6, one int64 column `ts` U[0, 10^6).
    strings_minmax   MIN(s) + MAX(s)
    strings_argmax   ARGMAX(s BY ts)
    int64_minmax / int64_argmax  the same shapes with an int64 value column in place of s, through the existing path.
  one_group_desc: 10^7 rows in one group, s strictly descending (8-digit decimals), MIN(s): every row improves the bound;
  int64_one_group_desc is the same with an int64 column.
  Rates are rows/s of the median step: a host clock around the call, which returns synchronised.
Parity: a seeded 10^6-row sample of the URL-like input (G = 10^3) on the GPU against the oracle's GROUP BY over the rank of
every string (equal ranks <=> equal strings, same order), one thread; that oracle run is also the CPU baseline.
Scalar leg (also the only leg with --scalar-only, which runs on a tree without string columns): N rows, two int64 keys
(U[0, 1000) x U[0, 8)), SUM + MIN + MAX + AVG of an int64 column through ytgpu_scan_filter_groupby_multi.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py
SLOT = 96
AGG_SUM, AGG_MIN, AGG_MAX, AGG_COUNT, AGG_AVG, AGG_ARGMIN, AGG_ARGMAX, AGG_FIRST = range(8)


def device_info():
    import torch
    power = None
    try:
        import pynvml as nv
        nv.nvmlInit()
        power = nv.nvmlDeviceGetPowerManagementLimit(nv.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        pass
    return torch.cuda.get_device_properties(0).name, power


def url_strings(n, g):
    """-> (heap, starts, lengths) on the device: URL-like strings in 96-byte slots."""
    import torch
    prefixes = [b"https://www.site%d.example.com/" % k for k in range(64)]
    width = max(len(p) for p in prefixes)
    ptab = torch.zeros((len(prefixes), SLOT), dtype=torch.uint8, device="cuda")
    for i, p in enumerate(prefixes):
        ptab[i, :len(p)] = torch.frombuffer(bytearray(p), dtype=torch.uint8).cuda()
    plen_tab = torch.tensor([len(p) for p in prefixes], device="cuda", dtype=torch.int64)
    heap = torch.empty((n, SLOT), dtype=torch.uint8, device="cuda")
    lengths = torch.empty(n, dtype=torch.int32, device="cuda")
    pos = torch.arange(SLOT, device="cuda")
    chunk = 1 << 23
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        h = torch.randint(0, len(prefixes), (b - a,), device="cuda", generator=g)
        plen = plen_tab[h]
        tail = torch.randint(97, 123, (b - a, SLOT), device="cuda", generator=g, dtype=torch.uint8)
        heap[a:b] = torch.where(pos[None, :] < plen[:, None], ptab[h], tail)
        lengths[a:b] = (plen + torch.randint(0, 49, (b - a,), device="cuda", generator=g)).to(torch.int32)
    assert width + 48 <= SLOT
    starts = torch.arange(n, device="cuda", dtype=torch.int64) * SLOT
    return heap.reshape(-1), starts, lengths


def decimal_strings(values):
    """8-digit zero-padded decimals on the device: string order == numeric order."""
    import torch
    x = values.clone()
    digits = torch.empty((len(values), 8), dtype=torch.uint8, device="cuda")
    for j in range(7, -1, -1):
        digits[:, j] = (48 + x % 10).to(torch.uint8)
        x = x // 10
    n = len(values)
    return digits.reshape(-1), torch.arange(n, device="cuda", dtype=torch.int64) * 8, torch.full((n,), 8, dtype=torch.int32, device="cuda")


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), min(ts), max(ts)


def leg(n, fn, steps, warmup):
    med, lo, hi = timed(fn, steps, warmup)
    return {"ms_median": round(med * 1e3, 3), "ms_min": round(lo * 1e3, 3), "ms_max": round(hi * 1e3, 3), "rows_per_s": n / med}


def scalar_leg(ctx, n, steps, warmup, g):
    import torch
    from ytsaurus_b200 import Column
    from ytsaurus_b200.rowset import EValueType as T
    k0 = torch.randint(0, 1000, (n,), device="cuda", generator=g)
    k1 = torch.randint(0, 8, (n,), device="cuda", generator=g)
    v = torch.randint(-10**9, 10**9, (n,), device="cuda", generator=g)
    keys = [Column(T.Int64, values=k0), Column(T.Int64, values=k1)]
    vals = [Column(T.Int64, values=v)]
    aggs = [(AGG_SUM, 0), (AGG_MIN, 0), (AGG_MAX, 0), (AGG_AVG, 0)]
    out = leg(n, lambda: ctx.scan_filter_groupby_multi(keys, vals, aggs, capacity=8000), steps, warmup)
    r = ctx.scan_filter_groupby_multi(keys, vals, aggs, capacity=8000)
    out["groups"] = len(r["count"])
    return out


def parity(ctx, g):
    """GPU vs the oracle over string ranks on a 10^6-row sample; -> (checks, mismatches, oracle seconds)."""
    import torch
    import oracle
    from ytsaurus_b200 import Column
    from ytsaurus_b200.rowset import EValueType as T
    m = 10**6
    heap, starts, lengths = url_strings(m, g)
    key = torch.randint(0, 1000, (m,), device="cuda", generator=g)
    ts = torch.randint(0, 10**6, (m,), device="cuda", generator=g)
    hb = heap.cpu().numpy().tobytes()
    ln = lengths.cpu().numpy()
    strs = [hb[i * SLOT:i * SLOT + int(ln[i])] for i in range(m)]
    uniq = sorted(set(strs))
    rank_of = {s: r for r, s in enumerate(uniq)}
    rank = np.asarray([rank_of[s] for s in strs], dtype=np.int64)
    kh, th = key.cpu().numpy(), ts.cpu().numpy()
    aggs_gpu = [(AGG_MIN, 1), (AGG_MAX, 1), (AGG_ARGMAX, 1, 0)]
    got = ctx.scan_filter_groupby_multi([Column(T.Int64, values=key)], [Column(T.Int64, values=ts)], aggs_gpu,
                                        string_columns=[(heap, starts, lengths, None)])
    t0 = time.perf_counter()
    want = oracle.groupby_multi([kh.view(np.uint64)], None, [rank.view(np.uint64), th.view(np.uint64), np.arange(m, dtype=np.uint64)], None,
                                [T.Int64, T.Int64, T.Int64], [(AGG_MIN, 0), (AGG_MAX, 0), (AGG_ARGMAX, 2, 1)])
    cpu_s = time.perf_counter() - t0
    bad = 0
    first = got["first_row"].cpu().numpy()
    bad += int((first != want["first_row"]).sum()) if len(first) == len(want["first_row"]) else 1
    rows = [v.cpu().numpy().view(np.int64) for v in got["values"]]
    if not bad:
        bad += int((rank[rows[0]] != want["values"][0].view(np.int64)).sum())
        bad += int((rank[rows[1]] != want["values"][1].view(np.int64)).sum())
        # MIN / MAX: the smallest row of the group that holds the value
        _, first_idx, inv = np.unique(kh * len(uniq) + rank, return_index=True, return_inverse=True)
        first_of = first_idx[inv]
        bad += int((first_of[rows[0]] != rows[0]).sum() + (first_of[rows[1]] != rows[1]).sum())
        bad += int((rows[2] != want["values"][2].view(np.int64)).sum())
    return {"rows": m, "groups": len(first), "checked": 4 * len(first), "mismatches": bad, "oracle_rows_per_s_1thread": m / cpu_s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scalar-only", action="store_true")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    import torch
    from ytsaurus_b200 import Column, GpuContext
    from ytsaurus_b200.rowset import EValueType as T
    assert torch.cuda.is_available(), "bench_groupby_strings.py needs a CUDA device"
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    ctx = GpuContext(0)
    n = args.rows
    name, power = device_info()
    line = {"bench": "groupby_strings", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps, "warmup": args.warmup}
    line["scalar_2keys_sum_min_max_avg"] = scalar_leg(ctx, n, args.steps, args.warmup, g)
    if not args.scalar_only:
        heap, starts, lengths = url_strings(n, g)
        ts = torch.randint(0, 10**6, (n,), device="cuda", generator=g)
        iv = torch.randint(-10**12, 10**12, (n,), device="cuda", generator=g)
        strings = [(heap, starts, lengths, None)]
        for groups in (10**3, 10**6):
            key = [Column(T.Int64, values=torch.randint(0, groups, (n,), device="cuda", generator=g))]
            vals = [Column(T.Int64, values=ts), Column(T.Int64, values=iv)]
            cap = groups

            def run(aggs, s=strings):
                return lambda: ctx.scan_filter_groupby_multi(key, vals, aggs, capacity=cap, group_count_hint=groups, string_columns=s)
            line[f"g{groups}"] = {
                "strings_minmax": leg(n, run([(AGG_MIN, 2), (AGG_MAX, 2)]), args.steps, args.warmup),
                "strings_argmax": leg(n, run([(AGG_ARGMAX, 2, 0)]), args.steps, args.warmup),
                "int64_minmax": leg(n, run([(AGG_MIN, 1), (AGG_MAX, 1)], ()), args.steps, args.warmup),
                "int64_argmax": leg(n, run([(AGG_ARGMAX, 1, 0)], ()), args.steps, args.warmup),
            }
            del key, vals
        del heap, starts, lengths, strings, ts, iv
        m = 10**7
        desc = torch.arange(m - 1, -1, -1, device="cuda", dtype=torch.int64)
        one = [Column(T.Int64, values=torch.zeros(m, dtype=torch.int64, device="cuda"))]
        s_desc = [decimal_strings(desc) + (None,)]
        line["one_group_desc"] = leg(m, lambda: ctx.scan_filter_groupby_multi(one, [], [(AGG_MIN, 0)], capacity=1, string_columns=s_desc),
                                     args.steps, args.warmup)
        r = ctx.scan_filter_groupby_multi(one, [], [(AGG_MIN, 0)], capacity=1, string_columns=s_desc)
        line["one_group_desc"]["min_row_ok"] = int(r["values"][0][0]) == m - 1
        line["int64_one_group_desc"] = leg(m, lambda: ctx.scan_filter_groupby_multi(one, [Column(T.Int64, values=desc)], [(AGG_MIN, 0)], capacity=1),
                                           args.steps, args.warmup)
        line["parity"] = parity(ctx, g)
    ctx.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
