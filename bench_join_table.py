#!/usr/bin/env python
"""bench_join_table.py — the join table on the GPU (ytgpu_join_table_build / ytgpu_join_table_probe): a dimension built once,
the fact side probed block by block, as a block map join runs it.

  python bench_join_table.py --steps K --warmup W [--rows N]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour; times are CUDA events
around the calls, after warm-up.  Legs (N = 10^8 primary rows by default):
  build          10^6 unique foreign int64 keys (a random half of [0, 2 * 10^6)), NULLS_NEVER_MATCH: the median time of
                 ytgpu_join_table_build (decode, assign, per-key counts and their scan, the stable sort of the foreign rows
                 by slot, the closing synchronisation)
  probe_<kind>_<block>  N primary int64 keys U[0, 2 * 10^6) against that table in blocks of 2^16, 2^20 and 2^24 rows, for
                 INNER, SEMI and ANTI, each block one ytgpu_join_table_probe with a capacity of the block's row count (the
                 keys are unique, so INNER has at most one pair per row): the median time per whole block, rows / s, and a
                 byte floor per block from the shapes: 8 B key read per row, plus for INNER 4 B slot + 8 B count written,
                 16 B of scan, 12 B of offset and slot read by the pair write and 8 B per pair written; for SEMI / ANTI 8 B
                 flag written, 16 B of scan, 8 B of offsets read by the listing and 4 B per listed row.  The table's own
                 random reads are not in the floor.  floor_fraction: that floor at 3.35 TB/s (H100 SXM data sheet) over the
                 measured time, a lower bound on the bandwidth share, not a roofline.
  star           the star leg of bench_join.py (N primary keys U[0, 10^6) against a shuffled 0 .. 10^6 - 1, INNER) as one
                 ytgpu_hash_join call against ytgpu_join_table_build + one ytgpu_join_table_probe, both with capacity N
String legs (ytgpu_join_table_build_strings / _probe_strings; --strings 0 leaves them out).  A key k of the legs above
becomes the 24 bytes "key-" + k in 20 zero-padded decimal digits, each row its own bytes in one device heap:
  build_string   the 10^6 foreign keys of build as strings: the median build time
  probe_string_<kind>_<block>  the N primary keys as strings, INNER and SEMI in blocks of 2^20 and 2^24 rows, as the probe
                 legs; floor_bytes: the int64 leg's floor plus, per row, the 24 string bytes, 12 B of start and length, and
                 the 8 B id written and read again
  probe_url_inner_16777216  INNER in blocks of 2^24 rows over keys of 20-120 bytes: key k is its 20-digit rendering
                 followed by filler up to a length of 20 + (k * 2654435761 mod 101) bytes; every row points at its key's
                 bytes in one heap of the 2 * 10^6 possible keys
  star_string    the star leg with its keys as strings: ytgpu_string_value_ids over foreign + primary and ytgpu_hash_join
                 over the ids (joint_ids) against the string table built and probed once (build_probe)
Parity: each probe kind's first 2^24-row block against numpy on a seeded sample of 10^5 rows (membership of the row's key
in the foreign keys, and the foreign row of each INNER pair), and star's two ways against each other (every pair) and
against numpy on the sample.  Each string probe leg's first block equals the int64 probe of the same keys (every row and
pair), and star_string's two ways give star's pairs.  One JSON line on stdout with the card's name and power limit; nothing is written to the
source tree.
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

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py
DATASHEET_HBM_BPS = 3.35e12
NO_ROW = 0xFFFFFFFF
BLOCKS = [1 << 16, 1 << 20, 1 << 24]


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


def render24(keys):
    """Non-negative int64 keys (a CUDA tensor) -> (heap, starts, lengths): row i is b"key-" + keys[i] in 20 decimal digits."""
    import torch
    n = keys.numel()
    heap = torch.empty((n, 24), dtype=torch.uint8, device="cuda")
    heap[:, :4] = torch.tensor(list(b"key-"), dtype=torch.uint8, device="cuda")
    pow10 = torch.tensor([10 ** (18 - i) for i in range(19)], dtype=torch.int64, device="cuda")
    for s in range(0, n, 1 << 24):  # the digits in chunks: (rows, 20) int64 temporaries
        k = keys[s:s + (1 << 24)]
        heap[s:s + k.numel(), 4] = 48  # keys < 10^19
        heap[s:s + k.numel(), 5:] = ((k[:, None] // pow10) % 10 + 48).to(torch.uint8)
    starts = torch.arange(n, device="cuda", dtype=torch.int64) * 24
    return heap.reshape(-1), starts, torch.full((n,), 24, dtype=torch.int32, device="cuda")


def time_blocks(fn, blocks, steps, warmup):
    """fn(start, rows) over every block, warmup + steps times -> (median ms of a whole block, the first call's outputs)."""
    import torch
    per_block, first = [], None
    for i in range(warmup + steps):
        spans = []
        for s, n in blocks:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = fn(s, n)
            b.record()
            spans.append((a, b, n))
            if i == 0 and s == 0:
                first = out
        torch.cuda.synchronize()
        if i >= warmup:
            per_block += [a.elapsed_time(b) for a, b, n in spans if n == blocks[0][1]]
    return statistics.median(per_block), first


def string_legs(ctx, args, line, parity, fkeys, pkeys, itable):
    import torch

    from ytsaurus_b200 import Column, capi
    from ytsaurus_b200.rowset import EValueType as T
    N, D = pkeys.numel(), fkeys.numel()
    fstr = render24(fkeys) + (None,)
    times = []
    for i in range(args.warmup + args.steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        t = ctx.join_table([], capi.JOIN_NULLS_NEVER_MATCH, string_keys=[fstr])
        b.record()
        b.synchronize()
        if i >= args.warmup:
            times.append(a.elapsed_time(b))
        t.close()
    ms = statistics.median(times)
    line["legs"]["build_string"] = {"foreign_rows": D, "key_bytes": 24, "median_ms": round(ms, 3), "rows_per_s": D / (ms / 1e3),
                                    "floor_bytes": D * (2 * (24 + 12) + 16)}
    heap, starts, lengths = render24(pkeys)
    stable = ctx.join_table([], capi.JOIN_NULLS_NEVER_MATCH, string_keys=[fstr])
    kinds = {"inner": capi.JOIN_INNER, "semi": capi.JOIN_SEMI}
    for kname, kind in kinds.items():
        for B in (1 << 20, 1 << 24):
            blocks = [(s, min(B, N - s)) for s in range(0, N, B)]
            ms, first = time_blocks(lambda s, n: stable.probe([], kind, capacity=n, out_mem=capi.MEM_DEVICE,
                                                               string_keys=[(heap, starts[s:s + n], lengths[s:s + n], None)]),
                                    blocks, args.steps, args.warmup)
            n0 = blocks[0][1]
            want = itable.probe([Column(T.Int64, values=pkeys[:n0].contiguous())], kind, capacity=n0, out_mem=capi.MEM_DEVICE)
            same = all(torch.equal(x, y) for x, y in zip(first, want)) if kind == capi.JOIN_INNER else torch.equal(first, want)
            parity.append(bool(same))
            listed = (first[0] if kind == capi.JOIN_INNER else first).numel()
            per_row = 8 + (12 + 16 + 12 if kind == capi.JOIN_INNER else 8 + 16 + 8) + 24 + 12 + 16
            floor = per_row * n0 + (8 if kind == capi.JOIN_INNER else 4) * listed
            line["legs"][f"probe_string_{kname}_{B}"] = {"block_rows": B, "blocks": len(blocks), "median_block_ms": round(ms, 4),
                                                         "rows_per_s": B / (ms / 1e3), "floor_bytes": floor,
                                                         "floor_fraction": floor / DATASHEET_HBM_BPS / (ms / 1e3), "same_as_int64": bool(same)}
    stable.close()
    del heap, starts, lengths
    # URL-like keys of 20-120 bytes: one heap row of 120 bytes per possible key, each row pointing at its key's
    dom = torch.arange(2 * D, device="cuda", dtype=torch.int64)
    ulen = (20 + (dom * 2654435761) % 101).to(torch.int32)
    uheap = (97 + (dom[:, None] + torch.arange(120, device="cuda")) % 26).to(torch.uint8)
    uheap[:, :20] = render24(dom)[0].reshape(-1, 24)[:, 4:]  # the 20 digits first: unique within every key's 20 or more bytes
    uheap = uheap.reshape(-1)
    ufor = (uheap, fkeys * 120, ulen[fkeys].contiguous(), None)
    B = 1 << 24
    with ctx.join_table([], capi.JOIN_NULLS_NEVER_MATCH, string_keys=[ufor]) as utable:
        blocks = [(s, min(B, N - s)) for s in range(0, N, B)]
        ustarts, ulens = pkeys * 120, ulen[pkeys].contiguous()
        ms, first = time_blocks(lambda s, n: utable.probe([], capi.JOIN_INNER, capacity=n, out_mem=capi.MEM_DEVICE,
                                                           string_keys=[(uheap, ustarts[s:s + n], ulens[s:s + n], None)]),
                                blocks, args.steps, args.warmup)
        n0 = blocks[0][1]
        want = itable.probe([Column(T.Int64, values=pkeys[:n0].contiguous())], capi.JOIN_INNER, capacity=n0, out_mem=capi.MEM_DEVICE)
        same = all(torch.equal(x, y) for x, y in zip(first, want))
        parity.append(bool(same))
        mean_len = float(ulens[:n0].float().mean())
        floor = round((8 + 12 + 16 + 12 + mean_len + 12 + 16) * n0 + 8 * first[0].numel())
        line["legs"][f"probe_url_inner_{B}"] = {"block_rows": B, "blocks": len(blocks), "mean_key_bytes": round(mean_len, 1),
                                                "median_block_ms": round(ms, 4), "rows_per_s": B / (ms / 1e3), "floor_bytes": floor,
                                                "floor_fraction": floor / DATASHEET_HBM_BPS / (ms / 1e3), "same_as_int64": bool(same)}


def star_string(ctx, args, line, parity, skeys, spk, want):
    """The star leg over 24-byte string keys: joint value ids + ytgpu_hash_join against the string table built and probed."""
    import torch

    from ytsaurus_b200 import Column, capi
    from ytsaurus_b200.rowset import EValueType as T
    N, D = spk.numel(), skeys.numel()
    fh, fs, fl = render24(skeys)
    ph, ps, pl = render24(spk)
    jh, js, jl = torch.cat([fh, ph]), torch.cat([fs, ps + fh.numel()]), torch.cat([fl, pl])  # foreign + primary, one column

    def joint_ids():
        ids, _ = ctx.string_value_ids(jh, js, jl)
        return ctx.hash_join([Column(T.Uint64, values=ids[D:])], [Column(T.Uint64, values=ids[:D])], capi.JOIN_INNER, capacity=N)

    def build_probe():
        with ctx.join_table([], capi.JOIN_NULLS_EQUAL, string_keys=[(fh, fs, fl, None)]) as t:
            return t.probe([], capi.JOIN_INNER, capacity=N, string_keys=[(ph, ps, pl, None)])
    leg = {"primary_rows": N, "foreign_rows": D, "key_bytes": 24}
    for name, fn in (("joint_ids", joint_ids), ("build_probe", build_probe)):
        times = []
        for i in range(args.warmup + args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = fn()
            b.record()
            b.synchronize()
            if i >= args.warmup:
                times.append(a.elapsed_time(b))
        same = all(torch.equal(x, y) for x, y in zip(out, want))
        parity.append(bool(same))
        leg[name + "_median_ms"] = round(statistics.median(times), 3)
        leg[name + "_same_pairs"] = bool(same)
        del out
    line["legs"]["star_string"] = leg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--strings", type=int, default=1)
    args = ap.parse_args()
    import torch

    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T

    assert torch.cuda.is_available(), "bench_join_table.py needs a CUDA device"
    name, power = device_info()
    ctx = GpuContext(0)
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    rng = np.random.default_rng(SEED)
    N, D = args.rows, 1_000_000
    col = lambda t: Column(T.Int64, values=t.contiguous())
    ev = lambda: torch.cuda.Event(enable_timing=True)
    line = {"bench": "join_table", "device": name, "power_limit_w": power, "rows": N, "steps": args.steps, "warmup": args.warmup,
            "legs": {}}
    parity = []

    # build
    fkeys = torch.randperm(2 * D, device="cuda", generator=g)[:D].contiguous()
    fcols = [col(fkeys)]
    times = []
    for i in range(args.warmup + args.steps):
        a, b = ev(), ev()
        a.record()
        table = ctx.join_table(fcols, capi.JOIN_NULLS_NEVER_MATCH)
        b.record()
        b.synchronize()
        if i >= args.warmup:
            times.append(a.elapsed_time(b))
        table.close()
    line["legs"]["build"] = {"foreign_rows": D, "median_ms": round(statistics.median(times), 3),
                             "rows_per_s": D / (statistics.median(times) / 1e3)}

    # probes
    pkeys = torch.randint(0, 2 * D, (N,), device="cuda", generator=g)
    member = torch.zeros(2 * D, dtype=torch.bool, device="cuda")
    member[fkeys] = True
    where = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
    where[fkeys] = torch.arange(D, device="cuda")
    table = ctx.join_table(fcols, capi.JOIN_NULLS_NEVER_MATCH)
    kinds = {"inner": capi.JOIN_INNER, "semi": capi.JOIN_SEMI, "anti": capi.JOIN_ANTI}
    for kname, kind in kinds.items():
        for B in BLOCKS:
            per_block = []
            blocks = [(s, min(B, N - s)) for s in range(0, N, B)]
            listed = 0
            for i in range(args.warmup + args.steps):
                spans = []
                for s, n in blocks:
                    a, b = ev(), ev()
                    a.record()
                    out = table.probe([col(pkeys[s:s + n])], kind, capacity=n, out_mem=capi.MEM_DEVICE)
                    b.record()
                    spans.append((a, b, n))
                    if i == 0 and B == BLOCKS[-1] and s == 0:  # parity on the first 2^24-row block
                        rows = np.unique(rng.integers(0, n, 100_000))
                        got_p = (out[0] if kind == capi.JOIN_INNER else out).cpu().numpy().view(np.uint32)
                        hit = member[pkeys[:n]].cpu().numpy()
                        want_listed = hit[rows] if kind != capi.JOIN_ANTI else ~hit[rows]
                        ok = np.array_equal(np.isin(rows, got_p), want_listed) and len(got_p) == int(
                            hit.sum() if kind != capi.JOIN_ANTI else n - hit.sum())
                        if kind == capi.JOIN_INNER:
                            got_f = out[1].cpu().numpy().view(np.uint32)
                            sel = rows[hit[rows]]
                            pos = np.searchsorted(got_p, sel)
                            ok = ok and np.array_equal(got_f[pos].astype(np.int64), where[pkeys[torch.from_numpy(sel).cuda()]].cpu().numpy())
                        parity.append(ok)
                    if i == args.warmup:
                        listed += (out[0] if kind == capi.JOIN_INNER else out).numel()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    per_block += [a.elapsed_time(b) for a, b, n in spans if n == B]
            ms = statistics.median(per_block)
            per_row = 8 + (12 + 16 + 12 if kind == capi.JOIN_INNER else 8 + 16 + 8)
            per_out = 8 if kind == capi.JOIN_INNER else 4
            floor = per_row * B + per_out * listed * B / N
            line["legs"][f"probe_{kname}_{B}"] = {"block_rows": B, "blocks": len(blocks), "median_block_ms": round(ms, 4),
                                                  "rows_per_s": B / (ms / 1e3), "listed_rows_per_block": round(listed * B / N),
                                                  "floor_bytes": round(floor),
                                                  "floor_fraction": floor / DATASHEET_HBM_BPS / (ms / 1e3)}
    if args.strings:
        string_legs(ctx, args, line, parity, fkeys, pkeys, table)
    table.close()
    del member, where

    # star: the one-shot call against build + one probe
    skeys = torch.randperm(D, device="cuda", generator=g)
    spk = torch.randint(0, D, (N,), device="cuda", generator=g)
    pc, fc = [col(spk)], [col(skeys)]

    def one_shot():
        return ctx.hash_join(pc, fc, capi.JOIN_INNER, capacity=N)

    def build_probe():
        with ctx.join_table(fc) as t:
            return t.probe(pc, capi.JOIN_INNER, capacity=N)
    star = {}
    outs = {}
    for leg, fn in (("one_shot", one_shot), ("build_probe", build_probe)):
        times = []
        for i in range(args.warmup + args.steps):
            a, b = ev(), ev()
            a.record()
            out = fn()
            b.record()
            b.synchronize()
            if i >= args.warmup:
                times.append(a.elapsed_time(b))
        outs[leg] = out
        star[leg + "_median_ms"] = round(statistics.median(times), 3)
    if args.strings:
        star_string(ctx, args, line, parity, skeys, spk, outs["one_shot"])
    same = all(torch.equal(x, y) for x, y in zip(outs["one_shot"], outs["build_probe"]))
    where = torch.empty(D, dtype=torch.int64, device="cuda")
    where[skeys] = torch.arange(D, device="cuda")
    rows = np.unique(rng.integers(0, N, 100_000))
    op = outs["one_shot"][0].cpu().numpy().view(np.uint32)
    of = outs["one_shot"][1].cpu().numpy().view(np.uint32)
    ok = len(op) == N and np.array_equal(op[rows], rows.astype(np.uint32)) and np.array_equal(
        of[rows].astype(np.int64), where[spk[torch.from_numpy(rows).cuda()]].cpu().numpy())
    parity += [same, bool(ok)]
    star.update({"primary_rows": N, "foreign_rows": D, "pairs": N, "same_pairs": same})
    line["legs"]["star"] = star
    line["parity"] = bool(all(parity))
    print(json.dumps(line), flush=True)
    ctx.close()
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
