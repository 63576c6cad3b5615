#!/usr/bin/env python
"""bench_groupby_table_strings.py — string-valued aggregates in the GROUP BY table on the GPU (ytgpu_groupby_table_*_strings):
MIN + MAX of a string folded block by block, against one ytgpu_scan_filter_groupby_multi_strings call over the same rows.

  python bench_groupby_table_strings.py --steps K --warmup W [--rows N] [--profile DIR]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour; times are CUDA events
around whole passes (every update and the result, or the one-shot call), median over the steps, after warm-up.  Legs
(N = 10^8 rows by default), each at 10^3 and 10^6 groups of an int64 key:
  url_<groups>         key U[0, groups), URL-like strings in 96-byte slots (bench_groupby_strings.url_strings): the
                       one-shot call, and the table fed in blocks of 2^20 rows
  descending_<groups>  the worst case for the table: key = row mod groups and strictly descending strings
                       ("https://example.com/" + 20 digits of 10^12 - row), so every update replaces every group's MIN
                       and appends all its bytes; the heap is compacted every few updates
Parity: each leg's table result equals its one-shot result bit for bit (groups, first rows, the selected rows and their
NULL flags), and the table's string bytes equal the input's at the selected rows (a 1000-group sample).  One JSON line
on stdout with the card's name and power limit; nothing is written to the source tree.  --profile DIR also records the
table over url_1000000 with torch.profiler, writes the Chrome trace to DIR and adds the CUDA time per kernel name per
update to the line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_groupby_strings import url_strings  # noqa: E402
from bench_groupby_table import SEED, host, profile, timed  # noqa: E402
from bench_join_table import device_info  # noqa: E402

BLOCK = 1 << 20


def descending(n):
    """-> (heap, starts, lengths) on the device: row i is "https://example.com/" + the 20 digits of 10^12 - i."""
    import torch
    width = 40
    heap = torch.empty((n, width), dtype=torch.uint8, device="cuda")
    heap[:, :20] = torch.tensor(list(b"https://example.com/"), dtype=torch.uint8, device="cuda")
    chunk = 1 << 24
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        k = 10**12 - torch.arange(a, b, device="cuda", dtype=torch.int64)
        for i in range(19, -1, -1):
            heap[a:b, 20 + i] = (k % 10 + 48).to(torch.uint8)
            k = k // 10
    return heap.reshape(-1), torch.arange(n, device="cuda", dtype=torch.int64) * width, torch.full((n,), width, dtype=torch.int32, device="cuda")


def same(got, ref, heap, starts, lengths):
    if len(host(got["count"])) != len(host(ref["count"])):
        return False
    ok = all((host(got[k]) == host(ref[k])).all() for k in ("count", "first_row"))
    ok = ok and (host(got["keys"][0]) == host(ref["keys"][0])).all()
    ok = ok and all((host(a) == host(b)).all() for a, b in zip(got["values"] + got["value_null"], ref["values"] + ref["value_null"]))
    g = len(host(got["count"]))
    sample = np.linspace(0, g - 1, min(g, 1000)).astype(np.int64)
    for j in range(2):
        rows = host(got["values"][j]).view(np.int64)[sample]
        gh, gs, gl, gn = (host(x) for x in got["string_values"][j])
        ok = ok and not gn.any()
        at = starts.new_tensor(rows)
        hs, hl = host(starts[at]), host(lengths[at])
        ok = ok and all(bytes(gh[int(gs[o]):int(gs[o]) + int(gl[o])]) == bytes(host(heap[int(hs[i]):int(hs[i]) + int(hl[i])]))
                        for i, o in enumerate(sample))
    return bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rows", type=int, default=10**8)
    ap.add_argument("--profile", default=None, help="directory for a torch.profiler trace of the url_1000000 table leg")
    args = ap.parse_args()
    import torch
    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T
    ctx = GpuContext(0)
    gen = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    n = args.rows
    aggs = [(capi.AGG_MIN, 0), (capi.AGG_MAX, 0)]  # column 0: the string value (no numeric value columns)
    legs, parity = {}, True
    updates = (n + BLOCK - 1) // BLOCK

    def table_pass(key, heap, starts, lengths, groups):
        def run():
            with ctx.groupby_table([T.Int64], 0, [], aggs, hint=groups, string_value_count=1) as t:
                for a in range(0, n, BLOCK):
                    b = min(n, a + BLOCK)
                    t.update([Column(T.Int64, values=key[a:b])], [], string_values=[(heap, starts[a:b], lengths[a:b], None)])
                return t.result(out_mem=capi.MEM_DEVICE)
        return run

    def one_shot(key, heap, starts, lengths, groups):
        return lambda: ctx.scan_filter_groupby_multi([Column(T.Int64, values=key)], [], aggs, group_count_hint=groups, capacity=groups,
                                                     string_columns=[(heap, starts, lengths, None)])

    for shape in ("url", "descending"):
        if shape == "url":
            heap, starts, lengths = url_strings(n, gen)
        else:
            heap, starts, lengths = descending(n)
        for groups in (10**3, 10**6):
            if shape == "url":
                key = torch.randint(0, groups, (n,), device="cuda", generator=gen, dtype=torch.int64)
            else:
                key = torch.arange(n, device="cuda", dtype=torch.int64) % groups
            one_ms, ref = timed(one_shot(key, heap, starts, lengths, groups), args.steps, args.warmup)
            ms, got = timed(table_pass(key, heap, starts, lengths, groups), args.steps, args.warmup)
            ok = same(got, ref, heap, starts, lengths)
            parity = parity and ok
            legs[f"{shape}_{groups}"] = {"one_shot_ms": round(one_ms, 3), "table_1048576_ms": round(ms, 3),
                                         "table_ms_per_update": round(ms / updates, 4), "parity": ok}
            if args.profile and shape == "url" and groups == 10**6:
                split = profile(table_pass(key, heap, starts, lengths, groups), args.profile)
                legs["profile_url_1000000_per_update"] = [dict(r, ms=round(r["ms"] / updates, 4)) for r in split]
            del key
        del heap, starts, lengths
        torch.cuda.empty_cache()

    name, power = device_info()
    print(json.dumps({"bench": "groupby_table_strings", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps,
                      "warmup": args.warmup, "legs": legs, "parity_ok": parity}))
    ctx.close()


if __name__ == "__main__":
    main()
