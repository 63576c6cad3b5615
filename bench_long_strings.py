#!/usr/bin/env python
"""bench_long_strings.py — rowset sort by string keys longer than the 256-byte normalised key.

  python bench_long_strings.py --steps K --warmup W [--rows N] [--dump-outputs DIR]

A rowset [key: string, payload: int64] of N rows (10^7 by default, generated on the device from a fixed seed) is sorted by
its key with ytgpu_sort_rowset in the DEVICE memory flavour.  Three inputs:
  url_like          one of 256 host prefixes of 24-40 bytes + a tail of U[0, 600] letters of a 16-letter alphabet; 10 % of
                    the rows copy the key of an earlier row.  The longest key is over 256 bytes: refinement rounds.
  shared_prefix     one fixed 1000-byte prefix + U[0, 64] random bytes (zero bytes included): refinement rounds.
  url_like_cut_200  url_like with the tails cut so that no key is longer than 200 bytes: the normalised-key path, the
                    reference point for keys that are wide but still fit.
Per input: rows/s (median step; a host clock around the call, which reads the unresolved row count back every round, so
the call ends synchronised), the refinement rounds and the rows each round sorted, and a parity check on the host (the
result is a permutation; ~10^5 sampled adjacent pairs are ordered by the oracle's comparator, equal keys in input order).
url_like also carries a CPU baseline: the oracle's SORT_STD (std::sort by the reference comparator, one thread) on its
first 10^6 rows.
Partition leg (`partition` per input): ytgpu_partition_rowset with the ordered partitioner (DEVICE, index + histogram)
for P = 8 and P = 1024 lower bounds.  Bound 0 is universal; bound j is the (j*m/P)-th key (prefix length 1, inclusive)
of a seeded sample of m = 10^5 rows sorted by the oracle.  Per P: rows/s (median step, a host clock around the call and a
device synchronise), `last_partition_key_words` (1: key words, 0: normalised keys), and parity of the sampled rows'
indices with the oracle's TOrderedPartitioner.  url_like also carries a CPU baseline: the oracle's partitioner on its
first 10^6 rows, one thread.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py


def gen_string_rowset(n, device, seed, prefixes, tail_max, alphabet, dup_frac=0.0, max_len=None):
    """-> (values [n, 2] as a uint8 tensor [n, 32], heap uint8 tensor) on the device.  Row i: key = prefixes[h_i] + a tail of
    U[0, tail_max] bytes drawn from `alphabet` (cut to max_len bytes in total); a `dup_frac` share of the rows copies the
    key of an earlier non-copied row; payload = i."""
    import torch
    from ytsaurus_b200.rowset import EValueType as T
    g = torch.Generator(device=device).manual_seed(seed)
    npre = len(prefixes)
    plen_tab = torch.tensor([len(p) for p in prefixes], device=device, dtype=torch.int64)
    width = max(len(p) for p in prefixes)
    ptab = torch.zeros((npre, width), dtype=torch.uint8, device=device)
    for i, p in enumerate(prefixes):
        ptab[i, : len(p)] = torch.frombuffer(bytearray(p), dtype=torch.uint8).to(device)
    alpha = torch.frombuffer(bytearray(alphabet), dtype=torch.uint8).to(device)
    h = torch.randint(0, npre, (n,), device=device, generator=g)
    plen = plen_tab[h]
    tlen = torch.randint(0, tail_max + 1, (n,), device=device, generator=g)
    if max_len is not None:
        tlen = torch.minimum(tlen, max_len - plen)
    klen = plen + tlen
    dup = torch.rand(n, device=device, generator=g) < dup_frac
    dup[0] = False
    klen_own = torch.where(dup, torch.zeros_like(klen), klen)
    off_own = torch.cumsum(klen_own, 0) - klen_own
    heap = torch.empty(int(klen_own.sum()) + 16, dtype=torch.uint8, device=device)
    chunk = 1 << 20
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        lens = klen_own[s:e]
        rid = torch.repeat_interleave(torch.arange(s, e, device=device), lens)
        pos = torch.arange(rid.numel(), device=device) - (torch.cumsum(lens, 0) - lens).repeat_interleave(lens)
        tail = alpha[torch.randint(0, len(alphabet), (rid.numel(),), device=device, generator=g)]
        pre = ptab[h[rid], torch.clamp(pos, max=width - 1)]
        heap[off_own[s] + torch.arange(rid.numel(), device=device)] = torch.where(pos < plen[rid], pre, tail)
    # a copied row takes the key of an earlier non-copied row
    own = torch.nonzero(~dup).squeeze(1)
    before = torch.searchsorted(own, torch.arange(n, device=device))  # non-copied rows before i
    pick = (torch.rand(n, device=device, generator=g) * before).to(torch.int64)
    src = torch.where(dup, own[torch.clamp(pick, max=own.numel() - 1)], torch.arange(n, device=device))
    vals = torch.zeros((n, 2, 4), dtype=torch.int32, device=device)  # (id | type << 16, length, data lo, data hi)
    vals[:, 0, 0] = T.String << 16
    vals[:, 0, 1] = klen[src].to(torch.int32)
    data = off_own[src]
    vals[:, 0, 2] = (data & 0xFFFFFFFF).to(torch.int32)
    vals[:, 0, 3] = (data >> 32).to(torch.int32)
    vals[:, 1, 0] = 1 | (T.Int64 << 16)
    vals[:, 1, 2] = torch.arange(n, device=device, dtype=torch.int32)
    return vals.view(torch.uint8).reshape(n, 32), heap


def parity_check(values_np, heap_np, perm, pairs=100_000, seed=SEED):
    """perm is a permutation; sampled adjacent pairs are ordered by the oracle's comparator, equal keys in input order."""
    import oracle
    n = len(perm)
    if not (np.bincount(perm.astype(np.int64), minlength=n) == 1).all():
        return {"ok": False, "reason": "not a permutation"}
    rng = np.random.default_rng(seed)
    js = rng.integers(0, n - 1, min(pairs, n - 1)) if n > 1 else np.zeros(0, np.int64)
    for j in js:
        a, b = int(perm[j]), int(perm[j + 1])
        c = oracle.compare_values(values_np[a, 0], values_np[b, 0], heap_np)
        if c > 0 or (c == 0 and a > b):
            return {"ok": False, "reason": f"positions {j}, {j + 1} out of order"}
    return {"ok": True, "pairs": int(len(js))}


def cpu_baseline(values_np, heap_np):
    import oracle
    _, sec = oracle.sort_rows(values_np, heap_np, 1, None, oracle.SORT_STD)
    return {"value": len(values_np) / sec, "unit": "rows/s", "cores": 1,
            "sample": f"first {len(values_np)} rows, the oracle's SORT_STD (std::sort by the reference comparator)"}


def partition_leg(ctx, vals, heap, vals_np, heap_np, steps, warmup, cpu_baseline_rows=0):
    """Ordered partitioning of the whole input for P = 8 and 1024 bounds taken from a sorted seeded sample."""
    import oracle
    from ytsaurus_b200 import capi
    from ytsaurus_b200.rowset import Rowset, VALUE_DTYPE
    n = len(vals_np)
    sample = vals_np[_sample_index(n, 100_000, SEED + 1)]
    m = len(sample)
    perm, _ = oracle.sort_rows(sample, heap_np, 1, None, oracle.SORT_STABLE)
    sorted_sample = sample[perm.astype(np.int64)]
    out = {}
    for P in (8, 1024):
        bvals = np.concatenate([np.zeros((1, 2), dtype=VALUE_DTYPE), sorted_sample[[(j * m) // P for j in range(1, P)]]])
        blen, binc = [0] + [1] * (P - 1), [1] * P
        spec = ctx._partition_spec(capi.PARTITION_ORDERED, P, key_columns=[dict(index=0, type=0x10)],
                                   bounds=Rowset(bvals, heap_np), bound_prefix_length=blen, bound_inclusive=binc)
        times, idx = [], None
        for step in range(warmup + steps):
            t0 = time.perf_counter()
            idx, _ = ctx.partition_rowset(vals, heap, spec)
            ctx.synchronize()
            if step >= warmup:
                times.append(time.perf_counter() - t0)
        r = {"partitions": P, "ms": [round(t * 1e3, 3) for t in times], "value": n / float(np.median(times)),
             "unit": "rows/s", "key_words": ctx.get_option("last_partition_key_words")}
        want, _ = oracle.partition_ordered(sample, heap_np, 1, None, bvals, heap_np, blen, binc)
        got = idx.cpu().numpy()[_sample_index(n, 100_000, SEED + 1)]
        r["parity_check"] = {"ok": bool((got == want).all()), "rows": int(m)}
        if cpu_baseline_rows:
            _, sec = oracle.partition_ordered(vals_np[:cpu_baseline_rows], heap_np, 1, None, bvals, heap_np, blen, binc)
            r["cpu_baseline"] = {"value": cpu_baseline_rows / sec, "unit": "rows/s", "cores": 1,
                                 "sample": f"first {cpu_baseline_rows} rows, the oracle's TOrderedPartitioner"}
        out[f"P{P}"] = r
    return out


def _sample_index(m, k, seed):
    """Sorted positions of a fixed seeded sample of k of m rows (every row when m <= k)."""
    if m <= k:
        return np.arange(m, dtype=np.int64)
    return np.sort(np.random.Generator(np.random.Philox(seed)).choice(m, k, replace=False)).astype(np.int64)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write a fixed sample of each input's permutation to DIR/<input>_perm_sample.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_strings.py needs a CUDA device (there is no CPU fallback)")
    from ytsaurus_b200 import GpuContext
    from ytsaurus_b200.rowset import VALUE_DTYPE
    device = torch.device("cuda", 0)
    ctx = GpuContext(0)
    n = args.rows
    rng = np.random.default_rng(SEED)
    letters = b"abcdefghijklmnop"
    hosts = [b"https://" + bytes(rng.choice(np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8), int(L) - 13)) + b".com/"
             for L in rng.integers(24, 41, 256)]
    shared = [bytes(rng.integers(0, 256, 1000, dtype=np.uint8))]
    inputs = {
        "url_like": dict(prefixes=hosts, tail_max=600, alphabet=letters, dup_frac=0.1),
        "shared_prefix": dict(prefixes=shared, tail_max=64, alphabet=bytes(range(256))),
        "url_like_cut_200": dict(prefixes=hosts, tail_max=600, alphabet=letters, dup_frac=0.1, max_len=200),
    }
    spec = [dict(index=0, type=0x10)]
    results = {}
    for name, kw in inputs.items():
        vals, heap = gen_string_rowset(n, device, SEED + len(results), **kw)
        torch.cuda.synchronize()
        max_len = int(vals.view(torch.int32).reshape(n, 8)[:, 1].max())
        times, perm = [], None
        for step in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            perm = ctx.sort_rowset(vals, heap, spec)
            ctx.synchronize()
            if step >= args.warmup:
                times.append(time.perf_counter() - t0)
        rounds = ctx.get_option("last_sort_refine_rounds")
        r = {"rows": n, "max_key_bytes": max_len, "heap_bytes": int(heap.numel()),
             "ms": [round(t * 1e3, 3) for t in times], "value": n / float(np.median(times)), "unit": "rows/s",
             "refine_rounds": rounds,
             "unresolved_rows_per_round": [ctx.get_option(f"last_sort_refine_rows.{i}") for i in range(rounds)]}
        perm_np = perm.cpu().numpy().view(np.uint32)
        vals_np = vals.cpu().numpy().reshape(-1).view(VALUE_DTYPE).reshape(n, 2)
        heap_np = heap.cpu().numpy()
        if name != "url_like_cut_200":
            r["parity_check"] = parity_check(vals_np, heap_np, perm_np)
        if name == "url_like" and not args.no_cpu_baseline:
            r["cpu_baseline"] = cpu_baseline(vals_np[: min(n, 1_000_000)], heap_np)
        r["partition"] = partition_leg(ctx, vals, heap, vals_np, heap_np, args.steps, args.warmup,
                                       min(n, 1_000_000) if name == "url_like" and not args.no_cpu_baseline else 0)
        if args.dump_outputs:
            os.makedirs(args.dump_outputs, exist_ok=True)
            np.save(os.path.join(args.dump_outputs, f"{name}_perm_sample.npy"), perm_np[_sample_index(n, 100_000, SEED)].astype(np.float64))
        results[name] = r
        del vals, heap, perm, vals_np, heap_np
        torch.cuda.empty_cache()
    name, power = device_info()
    line = {"metric": "rows/s sorted (rowset [string key > 256 B, int64], ytgpu_sort_rowset DEVICE)",
            "value": results["url_like"]["value"], "unit": "rows/s", "config": {"rows": n, "steps": args.steps, "warmup": args.warmup},
            "device": name, "power_limit_w": power,
            "parity_check": all(r.get("parity_check", {"ok": True})["ok"] and
                                all(p["parity_check"]["ok"] for p in r["partition"].values()) for r in results.values()),
            "inputs": results}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
