"""What one replica exchange of a sharded map costs on the bench workload (Merged, 640x480 room scans, 0.05 m
voxels): W ranks as W engines on one GPU, each rank's calls on a thread of its own (sharded.LocalAllGather
stands in for NCCL), an exchange after every scan.  Per exchange it reports the blocks and bytes received,
the time of ShardedLayer.exchange (device gather + all-gather + device upload; every call ends synchronised,
so the host clock measures the device work) with the all-gather's share, and the same for the host path
ShardedLayer.sync_replicas (mirror to host, host gather, upload from host) run on the same blocks.
The GPU's name and power limit are read in the same run.  WORLD (2), SCANS (12), WARM (2) set the size."""
import json
import os
import subprocess
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import voxblox_b200 as vb  # noqa: E402
from voxblox_b200 import scenes, sharded  # noqa: E402


class TimedGather:
    """A rank's all-gather with its time (synchronised on both ends) added to `spent`."""

    def __init__(self, inner):
        self.inner, self.spent = inner, 0.0

    def __call__(self, out, inp):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        self.inner(out, inp)
        torch.cuda.synchronize()
        self.spent += time.perf_counter() - t0


def host_all_gather(world):
    """sharded.all_gather_blocks for W threads of one process (host arrays, as sync_replicas hands them)."""
    parts, barrier = [None] * world, threading.Barrier(world)
    local = threading.local()

    def gather(indices, voxels, group=None):
        parts[local.rank] = (np.asarray(indices).reshape(-1, 3), np.asarray(voxels))
        barrier.wait()
        idx = np.concatenate([p[0] for p in parts])
        vox = np.concatenate([p[1].view(np.uint8).reshape(len(p[0]), -1) for p in parts])
        counts = np.array([len(p[0]) for p in parts])
        barrier.wait()
        return idx, vox, counts

    return gather, local


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    world = int(os.environ.get("WORLD", "2"))
    n_scans = int(os.environ.get("SCANS", "12"))
    warm = int(os.environ.get("WARM", "2"))
    scans = scenes.generate_parallel(scenes.c3_room_scan, range(n_scans))
    cfg = vb.TsdfIntegratorConfig(default_truncation_distance=0.2, integrator_threads=1)
    gather = sharded.LocalAllGather(world)
    ranks = []
    for r in range(world):
        layer = vb.Layer(0.05, 16, engine_options=sharded.shard_options(r, world, max_blocks=16384))
        integ = vb.TsdfIntegratorFactory.create("merged", cfg, layer)
        timed = TimedGather(gather.rank(r))
        ranks.append((layer, integ, sharded.ShardedLayer(layer, all_gather=timed), timed))
    host_gather, local = host_all_gather(world)
    sharded.all_gather_blocks = host_gather  # sync_replicas' collective, in process

    def run_rank(r, fn):
        local.rank = r
        t0 = time.perf_counter()
        out = fn()
        return out, time.perf_counter() - t0

    rows = []
    with ThreadPoolExecutor(world) as ex:
        for i, s in enumerate(scans):
            for _, integ, _, _ in ranks:
                integ.integratePointCloud((s[2], s[3]), s[0], s[1])
            for _, _, _, t in ranks:
                t.spent = 0.0
            res = list(ex.map(lambda r: run_rank(r, ranks[r][2].exchange), range(world)))
            ex_ms = 1e3 * max(t for _, t in res)
            ag_ms = 1e3 * max(t.spent for *_, t in ranks)
            stats = [ranks[r][2].last_exchange for r in range(world)]
            res_h = list(ex.map(lambda r: run_rank(r, ranks[r][2].sync_replicas), range(world)))
            host_ms = 1e3 * max(t for _, t in res_h)
            if i < warm:
                continue
            rows.append(dict(scan=i, blocks_received=sum(st["received"] for st in stats),
                             bytes_received=sum(st["bytes"] for st in stats), exchange_ms=round(ex_ms, 3),
                             exchange_all_gather_ms=round(ag_ms, 3),
                             sync_replicas_blocks_received=int(sum(b for b, _ in res_h)),
                             sync_replicas_ms=round(host_ms, 3)))
            print(json.dumps(rows[-1]), flush=True)
    summary = dict(gpu=gpu_identity(), world=world, scans=len(rows), workload="merged 640x480 room, 0.05 m voxels",
                   ranks="W engines on one GPU, in-process all-gather",
                   median_exchange_ms=float(np.median([r["exchange_ms"] for r in rows])),
                   median_sync_replicas_ms=float(np.median([r["sync_replicas_ms"] for r in rows])),
                   median_blocks_received=float(np.median([r["blocks_received"] for r in rows])),
                   median_bytes_received=float(np.median([r["bytes_received"] for r in rows])))
    print(json.dumps(summary), flush=True)
    out_dir = os.environ.get("OUT_DIR")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "shard_exchange_probe.json"), "w") as f:
            json.dump(dict(summary=summary, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
