#!/usr/bin/env python
"""bench_join.py — the hash JOIN on the GPU (ytgpu_hash_join) and the star-join query it serves.

  python bench_join.py --steps K --warmup W [--rows N]

All inputs are generated on the device from a fixed seed and passed in the DEVICE memory flavour.  Legs (N = 10^8 primary
rows by default):
  star            N primary int64 keys U[0, 10^6); 10^6 foreign rows with unique keys (a shuffled 0 .. 10^6 - 1): INNER,
                  N pairs
  half_miss_left  the same primary keys; 5 * 10^5 foreign rows, a random half of the range: LEFT, N pairs
  zipf            Zipf(1.1) primary keys over the 10^6 foreign keys of star (hot keys scattered over the range): INNER
  fanout          10^6 primary rows against 10^6 foreign rows, both U[0, 10^4): INNER, ~10^8 pairs (the output-bound leg)
  sorted_partial  star's primary keys sorted; 2 * 10^4 foreign rows with the keys of the first and last 1 % of the range:
                  INNER, ~2 * 10^6 pairs and one run of ~0.98 N primary rows without pairs (a sorted fact table against a
                  dimension that covers part of its key range)
  two_keys        two int64 key columns U[0, 1000) each; 10^6 foreign rows holding every pair once: INNER, N pairs
  star_groupby    star's join, a gather of one foreign column (region U[0, 100)), a gather of a primary column (amount) and
                  GROUP BY region with SUM(amount): SELECT d.region, sum(f.amount) FROM f JOIN d ON f.k = d.id GROUP BY
                  d.region, end to end
  snowflake_groupby  the evaluator's device call sequence for SELECT r.name, sum(f.amount) FROM f JOIN u ON f.user_id =
                  u.id JOIN r ON u.region_id = r.id GROUP BY r.name: N facts with user ids U[0, 10^6); 10^6 users with
                  unique ids and a region id U[0, 10^3); 10^3 regions with a string name.  Join, a gather of the users'
                  region id at the joined rows (clause 2's key), join, composition of the two row maps (gathers of the
                  maps as UINT64 columns), the final gathers (amount through the facts' map, the name through the regions'),
                  the name's string ids and GROUP BY them with SUM(amount)
Each leg reports the median call time (CUDA events around the call, after warm-up), primary rows / s, the time of timer
class 11 (build, probe, pair write and gathers; the stable sort of the foreign rows times itself under the sort classes)
and a byte floor computed from the shapes: 8 B per key column and row read on both sides, 8 B per pair written, and
40 B per primary row of slot and count traffic (probe: 4 B slot + 8 B count written; scan: 8 B read + 8 B written; pair
write: 8 B offset + 4 B slot read).  floor_fraction is that floor at 3.35 TB/s (the H100 SXM data sheet) over the measured
time: a lower bound on the share of bandwidth the call uses, not a roofline.
Parity: every leg checks a seeded sample of primary rows (10^6 rows; 10^4 for fanout, whose rows carry ~100 pairs each)
against a numpy reference (the foreign rows of each sampled row's key in ascending order, or NO_ROW), and star_groupby its
sums (and snowflake_groupby its sums by region name) against torch's index_add over all rows.  The project has no CPU port of the reference's JoinOpHelper, so there is no
CPU baseline and the line says so.  One JSON line on stdout, with the card's name and power limit; nothing is written to
the source tree.
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


def ranges(starts, counts):
    """Concatenation of [starts[i], starts[i] + counts[i])."""
    total = int(counts.sum())
    offs = np.cumsum(counts) - counts
    return np.repeat(starts - offs, counts) + np.arange(total, dtype=np.int64)


def check_sample(p_code, f_code, out_p, out_f, left, sample, rng):
    """The pairs of `sample` random primary rows against the numpy reference.  p_code / f_code: int64 key codes (one per
    row, equal iff the key tuples are equal) on the device."""
    import torch
    P = p_code.numel()
    rows = np.unique(rng.integers(0, P, sample))
    gp = out_p.cpu().numpy().view(np.uint32).astype(np.int64)
    gf = out_f.cpu().numpy().view(np.uint32)
    lo, hi = np.searchsorted(gp, rows, "left"), np.searchsorted(gp, rows, "right")
    fc = f_code.cpu().numpy()
    order = np.argsort(fc, kind="stable")
    fs = fc[order]
    pc = p_code[torch.from_numpy(rows).cuda()].cpu().numpy()
    l, r = np.searchsorted(fs, pc, "left"), np.searchsorted(fs, pc, "right")
    n = r - l
    if left:
        want_counts = np.maximum(n, 1)
        want = np.full(int(want_counts.sum()), NO_ROW, np.uint32)
        hit = np.repeat(n > 0, want_counts)
        want[hit] = order[ranges(l[n > 0], n[n > 0])]
    else:
        want_counts = n
        want = order[ranges(l, n)].astype(np.uint32)
    got_counts = hi - lo
    ok = np.array_equal(got_counts, want_counts) and np.array_equal(gf[ranges(lo, got_counts)], want)
    return bool(ok), int(rows.size)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    from ytsaurus_b200 import Column, GpuContext, capi
    from ytsaurus_b200.rowset import EValueType as T

    assert torch.cuda.is_available(), "bench_join.py needs a CUDA device"
    name, power = device_info()
    ctx = GpuContext(0)
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    rng = np.random.default_rng(SEED)
    N, D = args.rows, 1_000_000
    col = lambda t: Column(T.Int64, values=t.contiguous())
    ri = lambda lo, hi, n: torch.randint(lo, hi, (n,), device="cuda", generator=g, dtype=torch.int64)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ctx.reset_timers()
        ctx.enable_timers(True)
        times = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = fn()
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        ctx.enable_timers(False)
        ms, _ = ctx.kernel_ms(capi.KC_JOIN)
        return out, statistics.median(times), ms / args.steps

    star_keys = torch.randperm(D, device="cuda", generator=g)
    pkeys = ri(0, D, N)
    u = torch.rand(N, device="cuda", generator=g, dtype=torch.float64)
    zipf_rank = torch.clamp(torch.floor((1.0 - u).pow(-1.0 / 0.1)) - 1, max=1e18).to(torch.int64) % D
    del u
    zipf_keys = star_keys[zipf_rank]
    del zipf_rank
    half_keys = torch.randperm(D, device="cuda", generator=g)[: D // 2]
    legs = {
        "star": ([pkeys], [star_keys], capi.JOIN_INNER, 1_000_000),
        "half_miss_left": ([pkeys], [half_keys], capi.JOIN_LEFT, 1_000_000),
        "zipf": ([zipf_keys], [star_keys], capi.JOIN_INNER, 1_000_000),
        "fanout": ([ri(0, 10_000, D)], [ri(0, 10_000, D)], capi.JOIN_INNER, 10_000),
    }
    # a primary table sorted by key against a dimension that covers the first and last 1 % of the key range: the pair
    # write crosses a run of ~0.98 N rows without pairs
    covered = torch.cat([torch.arange(0, D // 100, device="cuda"), torch.arange(D - D // 100, D, device="cuda")])
    legs["sorted_partial"] = ([torch.sort(pkeys).values], [covered[torch.randperm(covered.numel(), device="cuda", generator=g)]],
                              capi.JOIN_INNER, 1_000_000)
    pair_perm = torch.randperm(D, device="cuda", generator=g)
    legs["two_keys"] = ([ri(0, 1000, N), ri(0, 1000, N)], [pair_perm // 1000, pair_perm % 1000], capi.JOIN_INNER, 1_000_000)
    line = {"bench": "join", "device": name, "power_limit_w": power, "rows": N, "steps": args.steps, "warmup": args.warmup,
            "cpu_baseline": "none: the project has no CPU port of JoinOpHelper", "legs": {}}
    for leg, (pk, fk, kind, sample) in legs.items():
        pcols, fcols = [col(t) for t in pk], [col(t) for t in fk]
        pairs = ctx.hash_join(pcols, fcols, kind, count_only=True)
        (op, of), ms, join_ms = timed(lambda: ctx.hash_join(pcols, fcols, kind, capacity=pairs))
        code = (lambda ks: ks[0] * 1000 + ks[1] if len(ks) == 2 else ks[0])
        ok, checked = check_sample(code(pk), code(fk), op, of, kind == capi.JOIN_LEFT, sample, rng)
        P, F = pk[0].numel(), fk[0].numel()
        floor = 8 * len(pk) * (P + F) + 8 * pairs + 40 * P
        line["legs"][leg] = {"primary_rows": P, "foreign_rows": F, "pairs": pairs, "median_ms": round(ms, 3),
                             "rows_per_s": P / (ms / 1e3), "join_class_ms": round(join_ms, 3), "floor_bytes": floor,
                             "floor_fraction": floor / DATASHEET_HBM_BPS / (ms / 1e3), "parity_rows": checked, "parity": ok}
        del op, of

    # star_groupby: the motivating query end to end
    region = ri(0, 100, D)
    amount = ri(-1000, 1000, N)
    pcols, fcols = [col(pkeys)], [col(star_keys)]
    rcol, acol = col(region), col(amount)

    def query():
        op, of = ctx.hash_join(pcols, fcols, capi.JOIN_INNER, capacity=N)
        r = ctx.gather_column(rcol, of)["column"]
        a = ctx.gather_column(acol, op)["column"]
        return ctx.scan_filter_groupby_multi([r], [a], [(capi.AGG_SUM, 0)], group_count_hint=100, capacity=128)
    res, ms, join_ms = timed(query)
    # every primary key has its one foreign row: the sum of region r is the amounts of the keys whose row holds r
    where = torch.empty(D, dtype=torch.int64, device="cuda")
    where[star_keys] = torch.arange(D, device="cuda")
    want = torch.zeros(100, dtype=torch.int64, device="cuda").index_add_(0, region[where[pkeys]], amount)
    keys = res["keys"][0].cpu().numpy().view(np.int64)
    sums = res["values"][0].cpu().numpy().view(np.int64)
    ok = len(keys) == 100 and bool((want.cpu().numpy()[keys] == sums).all())
    floor = 8 * (N + D) + 8 * N + 40 * N + 2 * (4 + 8) * N + 8 * N  # join + two gathers (row in, value out) + the GROUP BY read
    line["legs"]["star_groupby"] = {"primary_rows": N, "foreign_rows": D, "pairs": N, "median_ms": round(ms, 3),
                                    "rows_per_s": N / (ms / 1e3), "join_class_ms": round(join_ms, 3), "floor_bytes": floor,
                                    "floor_fraction": floor / DATASHEET_HBM_BPS / (ms / 1e3), "parity_rows": N, "parity": ok}

    # snowflake_groupby: two clauses, the second keyed on a column of the first clause's table
    R = 1000
    user_region = ri(0, R, D)
    region_ids = torch.randperm(R, device="cuda", generator=g)
    names = [b"region-%04d" % i for i in region_ids.tolist()]
    name_heap = torch.tensor(list(b"".join(names)), dtype=torch.uint8, device="cuda")
    name_lengths = torch.tensor([len(x) for x in names], dtype=torch.int32, device="cuda")
    name_starts = (torch.cumsum(name_lengths.to(torch.int64), 0) - name_lengths.to(torch.int64)).contiguous()
    ucol, rcol = col(user_region), col(region_ids)
    wide = lambda rows: Column(T.Uint64, values=rows.to(torch.int64))  # a row map as a UINT64 column
    narrow = lambda gathered: gathered["values"].to(torch.int32)

    def snowflake():
        p1, f1 = ctx.hash_join(pcols, fcols, capi.JOIN_INNER, capacity=N)
        key = ctx.gather_column(ucol, f1)["column"]
        pairs = ctx.hash_join([key], [rcol], capi.JOIN_INNER, count_only=True)
        p2, f2 = ctx.hash_join([key], [rcol], capi.JOIN_INNER, capacity=pairs)
        fact_map = narrow(ctx.gather_column(wide(p1), p2))
        narrow(ctx.gather_column(wide(f1), p2))  # the users' map, composed as the evaluator composes every earlier map
        amount_col = ctx.gather_column(acol, fact_map)["column"]
        _, starts, lengths, nulls = ctx.gather_string_column(name_heap, name_starts, name_lengths, None, f2)
        ids, _ = ctx.string_value_ids(name_heap, starts, lengths, nulls)
        res = ctx.scan_filter_groupby_multi([Column(T.Uint64, values=ids.view(torch.int64))], [amount_col], [(capi.AGG_SUM, 0)],
                                            group_count_hint=R, capacity=2 * R)
        return res, starts, lengths
    (res, starts, lengths), ms, join_ms = timed(snowflake)
    # every fact has its user and every user its region: the sum of region id r is the amounts of the facts whose user's
    # region is r
    want = torch.zeros(R, dtype=torch.int64, device="cuda").index_add_(0, user_region[where[pkeys]], amount).cpu().numpy()
    heap = bytes(name_heap.cpu().numpy())
    first = res["keys"][0].cpu().numpy().view(np.int64)
    got_starts, got_lengths = starts.cpu().numpy()[first], lengths.cpu().numpy()[first]
    sums = res["values"][0].cpu().numpy().view(np.int64)
    got = {int(heap[s:s + n].split(b"-")[1]): int(v) for s, n, v in zip(got_starts, got_lengths, sums)}
    present = np.unique(user_region.cpu().numpy())
    ok = len(got) == len(first) == present.size and all(got.get(int(r)) == int(want[r]) for r in present)
    # per fact row: both joins as the other legs count them, the key gather, the amount gather (4 B row in, 8 B out each),
    # two map compositions (4 B row + 8 B map value in, 8 B out each), the name gather (4 B row in, 13 B out), the string ids
    # (13 B in, 9 B out) and the GROUP BY read (16 B); the dimension-sized terms of the builds
    floor = 8 * (D + R) + (8 + 8 + 40) * 2 * N + 2 * 12 * N + 2 * 20 * N + 17 * N + 22 * N + 16 * N
    line["legs"]["snowflake_groupby"] = {"primary_rows": N, "foreign_rows": [D, R], "pairs": N, "median_ms": round(ms, 3),
                                         "rows_per_s": N / (ms / 1e3), "join_class_ms": round(join_ms, 3), "floor_bytes": floor,
                                         "floor_fraction": floor / DATASHEET_HBM_BPS / (ms / 1e3), "parity_rows": N, "parity": ok}
    line["parity"] = all(v["parity"] for v in line["legs"].values())
    print(json.dumps(line), flush=True)
    ctx.close()
    return 0 if line["parity"] else 1


if __name__ == "__main__":
    sys.exit(main())
