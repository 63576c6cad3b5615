#!/usr/bin/env python
"""bench_groupby_table.py — the GROUP BY table on the GPU (ytgpu_groupby_table_*): rows folded block by block against the
one-shot ytgpu_scan_filter_groupby_multi over the same rows.

  python bench_groupby_table.py --steps K --warmup W [--rows N]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour; times are CUDA events
around whole passes (every update and the result, or the one-shot call), median over the steps, after warm-up.  Legs
(N = 10^8 rows by default):
  numeric_<groups>  an int64 key U[0, groups) for groups = 10^3 and 10^6, SUM + COUNT + MIN + AVG over an int64 value:
                    the one-shot call, and the table fed in blocks of 2^16, 2^20 and 2^24 rows (time per whole input and
                    per update)
  tuple_<groups>    the same with a two-key tuple (key, key mod 7 as a double), blocks of 2^20 rows
  yql_single_key_<groups>  the YQL single-key BlockCombineHashed shape (host/tests/block_combine_bench.cpp, built with
                    the host adapters): N rows of an int64 key and value, SUM + COUNT, fed in Arrow batches of 2^20 rows to
                    the existing partial-states adapter and to the GROUP BY table adapter (staging
                    BlockCombineHashedKeysStageRows rows per update); host wall time of all batches plus Finish
  string_<groups>   N / 4 rows of a URL-like string key of 40-120 bytes ("https://example.com/" + 20 digits of the key,
                    padded by a filler that depends on the key), 10^3 and 10^6 distinct values: the one-shot call over
                    ytgpu_string_value_ids against the table fed in blocks of 2^20 rows
Parity: each leg's table result equals its one-shot result: groups, first rows, keys and COUNT(*) bit for bit, SUM /
COUNT / MIN bit for bit, AVG within 1e-9 relative (the header lets double sums add in any order).  The string legs
compare the table's string keys with the bytes at each group's first row.  One JSON line on stdout with the card's name and
power limit; nothing is written to the source tree.  --profile DIR also records the table over the 10^6-group input in
2^20-row blocks with torch.profiler, writes the Chrome trace to DIR and adds the CUDA time per kernel name to the line.
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
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_join_table import device_info  # noqa: E402

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py
BLOCKS = [1 << 16, 1 << 20, 1 << 24]


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), out


def host(x):
    import torch
    return x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def same(got, ref, avg_index=None):
    if len(host(got["count"])) != len(host(ref["count"])):
        return False
    ok = all((host(got[k]) == host(ref[k])).all() for k in ("count", "first_row"))
    ok = ok and all((host(a) == host(b)).all() for a, b in zip(got["keys"], ref["keys"]))
    for i, (a, b) in enumerate(zip(got["values"], ref["values"])):
        if i == avg_index:
            ok = ok and np.allclose(host(a).view(np.float64), host(b).view(np.float64), rtol=1e-9, equal_nan=True)
        else:
            ok = ok and (host(a) == host(b)).all()
    return bool(ok)


def profile(run, out_dir):
    """One pass of `run` under torch.profiler: the Chrome trace into out_dir, and CUDA ms per kernel name (top 12)."""
    import torch
    from torch.profiler import ProfilerActivity
    os.makedirs(out_dir, exist_ok=True)
    run()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, "groupby_table_1048576.json"))
    rows = []
    for e in prof.key_averages():
        dev = getattr(e, "device_time_total", None)
        if dev is None:
            dev = getattr(e, "cuda_time_total", 0)
        if dev and e.key and not e.key.startswith("ProfilerStep"):
            rows.append((dev / 1e3, e.count, e.key))
    rows.sort(reverse=True)
    return [{"kernel": k[:80], "ms": round(ms, 3), "calls": c} for ms, c, k in rows[:12]]


def urls(keys):
    """int64 keys (CUDA) -> (heap, starts, lengths): "https://example.com/" + the key in 20 digits + (k * 2654435761) mod 81
    bytes of filler, 40 to 120 bytes in all."""
    import torch
    n = keys.numel()
    width = 121
    heap = torch.full((n, width), ord("x"), dtype=torch.uint8, device="cuda")
    prefix = torch.tensor(list(b"https://example.com/"), dtype=torch.uint8, device="cuda")
    heap[:, :20] = prefix
    k = keys.clone()
    for i in range(19, -1, -1):
        heap[:, 20 + i] = (k % 10 + 48).to(torch.uint8)
        k = k // 10
    lengths = (40 + (keys * 2654435761) % 81).to(torch.int32)
    starts = torch.arange(n, device="cuda", dtype=torch.int64) * width
    return heap.reshape(-1), starts, lengths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rows", type=int, default=10**8)
    ap.add_argument("--profile", default=None, help="directory for a torch.profiler trace of the 2^20-row table leg")
    args = ap.parse_args()
    import torch
    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T
    ctx = GpuContext(0)
    gen = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    n = args.rows
    value = torch.randint(-10**6, 10**6, (n,), device="cuda", generator=gen, dtype=torch.int64)
    aggs = [(capi.AGG_SUM, 0), (capi.AGG_COUNT, 0), (capi.AGG_MIN, 0), (capi.AGG_AVG, 0)]
    legs, parity = {}, True

    def table_pass(key_types, key_cols, nstr, str_cols, vals, block, hint):
        def run():
            with ctx.groupby_table(key_types, nstr, [T.Int64], aggs, hint=hint) as t:
                rows = vals.numel()
                for a in range(0, rows, block):
                    b = min(rows, a + block)
                    t.update([Column(tp, values=c[a:b]) for tp, c in zip(key_types, key_cols)], [Column(T.Int64, values=vals[a:b])],
                             string_keys=[(h, s[a:b], ln[a:b], None) for h, s, ln in str_cols])
                return t.result(out_mem=capi.MEM_DEVICE)
        return run

    for groups in (10**3, 10**6):
        key = torch.randint(0, groups, (n,), device="cuda", generator=gen, dtype=torch.int64)
        one_ms, ref = timed(lambda: ctx.scan_filter_groupby_multi([Column(T.Int64, values=key)], [Column(T.Int64, values=value)], aggs,
                                                                  group_count_hint=groups), args.steps, args.warmup)
        leg = {"one_shot_ms": round(one_ms, 3)}
        for block in BLOCKS:
            ms, got = timed(table_pass([T.Int64], [key], 0, [], value, block, groups), args.steps, args.warmup)
            updates = (n + block - 1) // block
            leg[f"table_{block}_ms"] = round(ms, 3)
            leg[f"table_{block}_ms_per_update"] = round(ms / updates, 4)
            ok = same(got, ref, 3)
            leg[f"table_{block}_parity"] = ok
            parity = parity and ok
        legs[f"numeric_{groups}"] = leg
        # tuple keys
        second = (key % 7).to(torch.float64).view(torch.int64)
        one_ms, ref = timed(lambda: ctx.scan_filter_groupby_multi([Column(T.Int64, values=key), Column(T.Double, values=second)],
                                                                  [Column(T.Int64, values=value)], aggs, group_count_hint=groups),
                            args.steps, args.warmup)
        ms, got = timed(table_pass([T.Int64, T.Double], [key, second], 0, [], value, 1 << 20, groups), args.steps, args.warmup)
        ok = same(got, ref, 3)
        parity = parity and ok
        legs[f"tuple_{groups}"] = {"one_shot_ms": round(one_ms, 3), "table_1048576_ms": round(ms, 3), "parity": ok}
        if args.profile and groups == 10**6:
            legs["profile_numeric_1000000_1048576"] = profile(table_pass([T.Int64], [key], 0, [], value, 1 << 20, groups), args.profile)
        del key, second

    exe = os.path.join(ROOT, "host", "block_combine_bench")
    r = subprocess.run([exe, str(n), str(1 << 20), str(max(args.steps, 1))], capture_output=True, text=True, check=True)
    yql = json.loads(r.stdout)
    for name, leg in yql["legs"].items():
        legs[name] = leg
        parity = parity and leg["parity"]

    ns = n // 4
    for groups in (10**3, 10**6):
        key = torch.randint(0, groups, (ns,), device="cuda", generator=gen, dtype=torch.int64)
        heap, starts, lengths = urls(key)
        vals = value[:ns]

        def one_shot():
            ids = ctx.string_value_ids(heap, starts, lengths)
            ids = ids[0] if isinstance(ids, tuple) else ids
            return ctx.scan_filter_groupby_multi([Column(T.Uint64, values=ids)], [Column(T.Int64, values=vals)], aggs, group_count_hint=groups)
        one_ms, ref = timed(one_shot, args.steps, args.warmup)
        ms, got = timed(table_pass([], [], 1, [(heap, starts, lengths)], vals, 1 << 20, groups), args.steps, args.warmup)
        first = host(ref["first_row"]).astype(np.int64)
        gh, gs, gl, _ = (host(x) for x in got["string_keys"][0])
        want_len = host(lengths)[first]
        ok = (len(gl) == len(first) and (gl.astype(np.int64) == want_len).all() and (host(got["first_row"]) == host(ref["first_row"])).all()
              and all((host(a) == host(b)).all() for a, b in zip(got["values"][:3], ref["values"][:3])))
        hh = host(heap)
        hs = host(starts)
        sample = np.linspace(0, len(first) - 1, min(len(first), 1000)).astype(np.int64)
        ok = ok and all(bytes(gh[int(gs[o]):int(gs[o]) + int(gl[o])]) == bytes(hh[int(hs[first[o]]):int(hs[first[o]]) + int(want_len[o])])
                        for o in sample)
        ok = bool(ok)
        parity = parity and ok
        legs[f"string_{groups}"] = {"rows": ns, "one_shot_value_ids_ms": round(one_ms, 3), "table_1048576_ms": round(ms, 3), "parity": ok}
        del key, heap, starts, lengths

    name, power = device_info()
    print(json.dumps({"bench": "groupby_table", "device": name, "power_limit_w": power, "rows": n, "steps": args.steps,
                      "warmup": args.warmup, "legs": legs, "parity_ok": parity}))
    ctx.close()


if __name__ == "__main__":
    main()
