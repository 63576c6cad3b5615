"""ORDER BY ... LIMIT on the GPU (ytgpu_order_rows): four legs, each result checked against numpy.

  sort_1e8_int64_limit100     10^8 rows ORDER BY one int64 LIMIT 100
  sort_1e7_int64desc_url      10^7 rows ORDER BY (int64 DESC over 1000 values, a URL-like string of 20..32 bytes) LIMIT 100
  groups_1e6_sum_desc_limit10 10^6 group sums (a GROUP BY's output) ORDER BY sum DESC LIMIT 10
  where_1pct_of_1e8           a 1 % WHERE row list over 10^8 rows, ORDER BY int64 LIMIT 1000

Each leg reports the median wall time of --steps calls after --warmup (the call synchronises its stream, so the host clock
covers the work), and a split of the call from the context's CUDA-event timers (medians of --steps more calls):
  materialise_ms      the kernel that writes the typed columns as the 16-byte rowset.  It is timed as key extraction (class
                      2), and so is the sort's own key normalisation, so it is class 2 of the call minus class 2 of a
                      ytgpu_sort_rowset of the same rowset with the same key spec (built here with torch), calls alternated
  key_normalise_ms    class 2 of that ytgpu_sort_rowset: the sort's key normalisation (and prefix chunk)
  sort_and_window_ms  the sort's other classes (digit passes, histograms, tails, gathers) and the window kernel, plus
                      key_normalise_ms
materialise_gbs is the materialisation's algorithmic bytes (per row: the item columns' bytes and the row list read, 16 B
per item written) over materialise_ms.  The checks recompute the window with numpy:
candidates at or past the window's threshold value, ordered stably by (key, row).  One JSON line on stdout, with the
card's name and power limit; nothing is written to the tree."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py


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


def top_stable(key, rows, limit):
    """The first `limit` of `rows` ordered stably by the uint64 `key` of each row (numpy)."""
    k = key[rows]
    if limit < len(rows):
        thr = np.partition(k, limit - 1)[limit - 1]
        sel = k <= thr
        rows, k = rows[sel], k[sel]
    return rows[np.lexsort((rows, k))][:limit]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch

    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T

    assert torch.cuda.is_available(), "bench_order.py needs a CUDA device"
    name, power = device_info()
    ctx = GpuContext(0)
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    rng = np.random.default_rng(SEED)
    N = args.rows
    legs = {}

    def rowset(items):
        """The rowset ytgpu_order_rows materialises: [(type, int64 payload tensor, lengths or None)] -> uint8 [n, 16 k]."""
        n = items[0][1].numel()
        words = torch.empty((n, 2 * len(items)), dtype=torch.int64, device="cuda")
        for k, (vtype, data, lengths) in enumerate(items):
            w0 = torch.full((n,), k | (int(vtype) << 16), dtype=torch.int64, device="cuda")
            if lengths is not None:
                w0 |= lengths.to(torch.int64) << 32
            words[:, 2 * k] = w0
            words[:, 2 * k + 1] = data
        return words.view(torch.uint8).reshape(n, 16 * len(items))

    def run(leg, call, check, values, heap, spec, read_bytes_per_row):
        for _ in range(args.warmup):
            call()
            ctx.sort_rowset(values, heap, spec)
        times = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            out = call()
            times.append((time.perf_counter() - t0) * 1e3)
        ctx.enable_timers(True)
        order_extract, sort_extract, rest = [], [], []
        for _ in range(args.steps):
            ctx.reset_timers()
            call()
            order_extract.append(ctx.kernel_ms(capi.KC_EXTRACT)[0])
            rest.append(sum(ctx.kernel_ms(c)[0] for c in (capi.KC_RADIX_PASS, capi.KC_GATHER, capi.KC_HISTOGRAM, capi.KC_PASS_SKIPPED)))
            ctx.reset_timers()
            ctx.sort_rowset(values, heap, spec)
            sort_extract.append(ctx.kernel_ms(capi.KC_EXTRACT)[0])
        ctx.enable_timers(False)
        normalise = statistics.median(sort_extract)
        materialise = statistics.median(order_extract) - normalise
        rows = values.shape[0]
        nbytes = rows * (read_bytes_per_row + values.shape[1])
        legs[leg] = {"ms": round(statistics.median(times), 3), "materialise_ms": round(materialise, 3),
                     "key_normalise_ms": round(normalise, 3), "sort_and_window_ms": round(statistics.median(rest) + normalise, 3),
                     "materialise_gbs": round(nbytes / (materialise * 1e6), 1) if materialise > 0 else None,
                     "ok": bool(check(out.cpu().numpy().view(np.uint32).astype(np.int64)))}

    # 1. 10^8 int64 rows, LIMIT 100
    a = torch.randint(-2**62, 2**62, (N,), device="cuda", generator=g, dtype=torch.int64)
    a_key = (a.cpu().numpy().view(np.uint64) ^ np.uint64(1 << 63))
    all_rows = np.arange(N, dtype=np.int64)
    empty_heap = torch.zeros(1, dtype=torch.uint8, device="cuda")
    run("sort_1e8_int64_limit100", lambda: ctx.order_rows([Column(T.Int64, values=a)], items=[(0, False, False)], limit=100),
        lambda got: np.array_equal(got, top_stable(a_key, all_rows, 100)),
        rowset([(T.Int64, a, None)]), empty_heap, [(0, 0, T.Int64, 0, 0)], 8)

    # 2. 10^7 rows by (int64 DESC over 1000 values, URL-like string)
    M = min(N, 10_000_000)
    b = torch.randint(0, 1000, (M,), device="cuda", generator=g, dtype=torch.int64)
    width = 32
    body = rng.integers(ord("a"), ord("e"), (M, width), dtype=np.uint8)  # four letters: long shared prefixes
    body[:, :15] = np.frombuffer(b"https://ex.com/", np.uint8)
    lengths = rng.integers(20, width + 1, M).astype(np.uint32)
    heap = torch.from_numpy(body.reshape(-1)).cuda()
    starts = torch.arange(0, M * width, width, device="cuda", dtype=torch.int64)
    lens = torch.from_numpy(lengths.view(np.int32)).cuda()
    nulls = torch.zeros(M, dtype=torch.uint8, device="cuda")
    b_np = b.cpu().numpy()

    def check_url(got):
        thr = np.sort(b_np)[::-1][99]
        cand = np.flatnonzero(b_np >= thr)
        strs = [bytes(body[i, :lengths[i]]) for i in cand]
        order = sorted(range(len(cand)), key=lambda j: (-b_np[cand[j]], strs[j], cand[j]))
        return np.array_equal(got, cand[order][:100])
    run("sort_1e7_int64desc_url", lambda: ctx.order_rows([Column(T.Int64, values=b)], [(heap, starts, lens, nulls)],
                                                          [(0, False, True), (0, True, False)], limit=100), check_url,
        rowset([(T.Int64, b, None), (T.String, starts, lens)]), heap, [(0, 0, T.Int64, 1, 0), (1, 0, T.String, 0, 0)], 8 + 8 + 4 + 1)

    # 3. 10^6 group sums ORDER BY sum DESC LIMIT 10
    G = 1_000_000
    keys = torch.randint(0, G, (M,), device="cuda", generator=g, dtype=torch.int64)
    vals = torch.randint(-1000, 1000, (M,), device="cuda", generator=g, dtype=torch.int64)
    sums = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, keys, vals)
    s_key = ~(sums.cpu().numpy().view(np.uint64) ^ np.uint64(1 << 63))  # descending
    run("groups_1e6_sum_desc_limit10", lambda: ctx.order_rows([Column(T.Int64, values=sums)], items=[(0, False, True)], limit=10),
        lambda got: np.array_equal(got, top_stable(s_key, np.arange(G, dtype=np.int64), 10)),
        rowset([(T.Int64, sums, None)]), empty_heap, [(0, 0, T.Int64, 1, 0)], 8)

    # 4. a 1 % WHERE row list over the 10^8 rows of leg 1
    sel = np.sort(rng.choice(N, N // 100, replace=False)).astype(np.uint32)
    sel_dev = torch.from_numpy(sel.view(np.int32)).cuda()
    run("where_1pct_of_1e8", lambda: ctx.order_rows([Column(T.Int64, values=a)], items=[(0, False, False)], rows=sel_dev, limit=1000),
        lambda got: np.array_equal(got, top_stable(a_key, sel.astype(np.int64), 1000)),
        rowset([(T.Int64, a[sel_dev.long()], None)]), empty_heap, [(0, 0, T.Int64, 0, 0)], 4 + 8)

    line = {"bench": "order", "device": name, "power_limit_w": power, "rows": N, "steps": args.steps, "warmup": args.warmup,
            "legs": legs, "ok": all(v["ok"] for v in legs.values())}
    print(json.dumps(line))
    ctx.close()
    return 0 if line["ok"] else 1


if __name__ == "__main__":
    sys.exit(main())
