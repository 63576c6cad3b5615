#!/usr/bin/env python
"""bench_peer_scatter.py — the streaming row exchange of the in-box shuffle (ytgpu_scatter_rows_to_peers) on one GPU.

  python bench_peer_scatter.py --steps K --warmup W [--rows N] [--parts 2,8,32]

N rows (10^8 by default) of 64 bytes and a uniform int32 partition index are generated on the device from a fixed seed;
every partition's slab is a slice of one local buffer, so the exchange runs the same kernels as the multi-GPU sort
(counting pass, scan of the [partition][tile] count matrix, destination-order scatter) without NVLink.  Each partition
count reports the median over the steps of:
  count_scan_ms  the library's KC_PARTITION timer: tile_count_kernel, the three scan launches and the totals check
  scatter_ms     the KC_SCATTER timer: scatter_stream_kernel
  call_ms        host clock around the whole call, which ends in a stream synchronise
After the timed steps the slabs are compared with the rows in stable partition order.
One JSON line on stdout, with the card's name and power limit.  Nothing is written to the source tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEED = 0x5954534155525553  # "YTSAURUS", as bench.py
ROW_BYTES = 64


def device_info():
    """Name, PCI bus id and power limit of the card the timing ran on (torch's cuda:0, which under CUDA_VISIBLE_DEVICES
    need not be nvidia-smi's index 0: the card is matched by UUID, or by bus id where nvidia-smi reports no UUID)."""
    import torch
    p = torch.cuda.get_device_properties(0)
    uuid = str(p.uuid).lower()
    bus_id = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    power = None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=uuid,pci.bus_id,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        for line in out.stdout.strip().splitlines():
            smi_uuid, bus, limit = (x.strip() for x in line.split(","))
            if smi_uuid.lower().endswith(uuid) or bus.upper() == bus_id:
                power = float(limit)
    except Exception:
        pass
    return p.name, bus_id, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--parts", default="2,8,32")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    parts_list = [int(p) for p in args.parts.split(",")]
    if any(not 1 <= p <= 32 for p in parts_list):
        ap.error("--parts must be in [1, 32]: the streaming exchange")
    import torch

    from ytsaurus_b200 import GpuContext, capi
    assert torch.cuda.is_available(), "bench_peer_scatter.py needs a CUDA device"
    n = args.rows
    g = torch.Generator(device="cuda").manual_seed(SEED & 0x7FFFFFFFFFFFFFFF)
    rows = torch.randint(0, 256, (n * ROW_BYTES,), dtype=torch.uint8, device="cuda", generator=g)
    dest = torch.empty_like(rows)
    ctx = GpuContext(0)
    ctx.enable_timers(True)
    results = {}
    for parts in parts_list:
        idx = torch.randint(0, parts, (n,), dtype=torch.int32, device="cuda", generator=g)
        counts = torch.bincount(idx, minlength=parts).cpu().tolist()
        starts = [0]
        for c in counts[:-1]:
            starts.append(starts[-1] + c)
        ptrs = [dest.data_ptr() + s * ROW_BYTES for s in starts]
        torch.cuda.synchronize()
        count_scan, scatter, call = [], [], []
        for step in range(args.warmup + args.steps):
            ctx.reset_timers()
            t0 = time.perf_counter()
            ctx.scatter_rows_to_peers(rows, ROW_BYTES, idx, counts, ptrs)
            t1 = time.perf_counter()
            if step >= args.warmup:
                count_scan.append(ctx.kernel_ms(capi.KC_PARTITION)[0])
                scatter.append(ctx.kernel_ms(capi.KC_SCATTER)[0])
                call.append((t1 - t0) * 1e3)
        order = torch.argsort(idx, stable=True)
        ok = bool(torch.equal(dest.view(n, ROW_BYTES), rows.view(n, ROW_BYTES)[order]))
        del order
        results[str(parts)] = {
            "count_scan_ms": round(statistics.median(count_scan), 4),
            "count_scan_range_ms": [round(min(count_scan), 4), round(max(count_scan), 4)],
            "scatter_ms": round(statistics.median(scatter), 4),
            "scatter_range_ms": [round(min(scatter), 4), round(max(scatter), 4)],
            "call_ms": round(statistics.median(call), 4),
            "slabs_match": ok,
        }
    ctx.close()
    name, bus_id, power = device_info()
    line = {"bench": "peer_scatter", "rows": n, "row_bytes": ROW_BYTES, "steps": args.steps, "device": name,
            "pci_bus_id": bus_id, "power_limit_w": power, "parts": results}
    print(json.dumps(line), flush=True)
    if not all(r["slabs_match"] for r in results.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
