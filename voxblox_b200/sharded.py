"""One map over the GPUs of a box: block-ownership sharding (BASELINE.json north_star, SURVEY.md
section 8e; DESIGN.md "multi-GPU").  One process per GPU, torch.distributed for the plumbing.

Every rank is handed EVERY scan and runs the ordinary integrators; the engine (created with
EngineOptions(rank=r, world_size=W)) applies only the voxel updates of the blocks rank r owns and
creates only those blocks.  Bundling, the reference's bundle order, the merge and the ray walk are
the same deterministic computation on every rank, so the ranks need no exchange while integrating:
the union of the W shards is the single-GPU map bit for bit (tests/test_sharded_gpu.py), every voxel
keeping the reference's one-thread update order.

Why no reduce: the reference's closest multi-map model is the layer merge of
voxblox/src/utils/voxel_utils.cc:9-22, which is associative only because it averages; the
integrator's clamp after every update (tsdf_integrator.cc:205-208) is not, so partial TSDF sums
from different ray ranges cannot be combined into the reference's result.  Ownership sharding keeps
every voxel's update chain on one GPU instead.

This module holds the host-side logic: the ownership function (mirrors vbx_block_owner), gathering
the shards into one block dictionary, and keeping read-only replicas of the other ranks' dirty blocks:
`exchange` moves them GPU to GPU (device gather, one all-gather of CUDA tensors, device upload), so
that the ESDF, the mesher and ICP of every rank see the whole map; `sync_replicas` is the older path
through host memory.
"""
from __future__ import annotations

import threading
from typing import Callable, Dict, Optional, Tuple

import numpy as np

from .api import (UPDATED_ESDF, UPDATED_MAP, UPDATED_MESH, UPDATED_MIRROR, EngineOptions, Layer,
                  VoxbloxError)

# the updated() bits a replica carries: what Block::updated().set() gives a block a scan touched
# (tsdf_integrator.cc:91-134), so incremental consumers on the receiving rank see it as the owner's would
REPLICA_BITS = UPDATED_MAP | UPDATED_MESH | UPDATED_ESDF


# ------------------------------------------------------------------ host logic (CPU-testable)
def block_owner(index, world: int) -> np.ndarray:
    """vbx_block_owner: rank owning block (bx, by, bz) = (bx + 2 by + 4 bz) mod world (non-negative)."""
    idx = np.asarray(index, dtype=np.int64).reshape(-1, 3)
    return ((idx[:, 0] + 2 * idx[:, 1] + 4 * idx[:, 2]) % int(world)).astype(np.int32)


def shard_options(rank: int, world: int, **kw) -> EngineOptions:
    """EngineOptions for rank `rank` of a `world`-way sharded map."""
    if not 0 <= rank < world:
        raise VoxbloxError("rank outside [0, world_size)")
    return EngineOptions(rank=rank, world_size=world, **kw)


def pack_blocks(indices: np.ndarray, voxels: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(M, 3) int32 indices and (M, vps^3) voxel records -> two contiguous byte arrays."""
    idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
    vox = np.ascontiguousarray(voxels)
    return idx.view(np.uint8).reshape(-1), vox.view(np.uint8).reshape(-1)


def all_gather_blocks(indices: np.ndarray, voxels: np.ndarray, group=None):
    """All ranks' (indices, voxels), rank after rank.  Variable block counts per rank: the counts
    travel first, then one padded all-gather (gloo on CPU tensors, NCCL on CUDA tensors)."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    nccl = dist.get_backend(group) == "nccl"
    dev = torch.device("cuda", torch.cuda.current_device()) if nccl else torch.device("cpu")
    idx_b, vox_b = pack_blocks(indices, voxels)
    m = int(np.asarray(indices).reshape(-1, 3).shape[0])
    per_block = int(vox_b.size // m) if m else int(voxels.dtype.itemsize * (voxels.shape[-1] if voxels.ndim > 1 else 0))
    meta = torch.tensor([m, per_block], dtype=torch.int64, device=dev)
    metas = torch.zeros(world * 2, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(metas, meta, group=group)
    metas = metas.cpu().numpy().reshape(world, 2)
    counts = metas[:, 0]
    per_block = int(metas[:, 1].max())
    cap = int(counts.max())
    out_idx, out_vox = [], []
    if cap == 0:
        return np.zeros((0, 3), np.int32), np.zeros((0,), np.uint8), counts
    send = torch.zeros(cap * (12 + per_block), dtype=torch.uint8, device=dev)
    if m:
        send[: m * 12] = torch.from_numpy(idx_b.copy()).to(dev)
        send[cap * 12: cap * 12 + m * per_block] = torch.from_numpy(vox_b.copy()).to(dev)
    recv = torch.zeros(world * send.numel(), dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(recv, send, group=group)
    recv = recv.cpu().numpy().reshape(world, -1)
    for r in range(world):
        c = int(counts[r])
        out_idx.append(recv[r, : c * 12].view(np.int32).reshape(c, 3))
        out_vox.append(recv[r, cap * 12: cap * 12 + c * per_block].reshape(c, per_block))
    return np.concatenate(out_idx), np.concatenate(out_vox), counts


def nccl_all_gather(group=None) -> Callable:
    """all_gather(out, inp): torch.distributed.all_gather_into_tensor over `group` (NCCL on CUDA tensors)."""
    import torch.distributed as dist

    return lambda out, inp: dist.all_gather_into_tensor(out, inp, group=group)


class LocalAllGather:
    """The all-gather of W ranks that are W threads of one process, each with its own engine (all on one
    GPU, or several): rank r calls `gather.rank(r)(out, inp)` from its thread, as it would call
    all_gather_into_tensor.  Lets a sharded map run without torch.distributed (tests, single-GPU
    measurement)."""

    def __init__(self, world: int, timeout: float = 300.0):
        self.world = world
        self._inputs = [None] * world
        self._barrier = threading.Barrier(world, timeout=timeout)

    def rank(self, r: int) -> Callable:
        import torch

        def gather(out, inp):
            self._inputs[r] = inp
            self._barrier.wait()
            torch.cat([p.to(out.device) for p in self._inputs], out=out)
            self._barrier.wait()  # (no rank replaces its input before every rank has read it)

        return gather


class ShardedLayer:
    """The block-sharded map as its callers see it.

    `layer` is this rank's shard (a Layer whose engine was created with shard_options).  `all_gather`
    (out, inp) is the collective exchange() uses, all_gather_into_tensor over `group` by default; with
    another one (LocalAllGather) rank and world come from the layer's engine options."""

    def __init__(self, layer: Layer, group=None, all_gather: Optional[Callable] = None):
        self.layer = layer
        self.group = group
        if all_gather is None:
            import torch.distributed as dist

            self.rank = dist.get_rank(group)
            self.world = dist.get_world_size(group)
            all_gather = nccl_all_gather(group)
        else:
            self.rank = int(layer.engine_options.rank)
            self.world = int(layer.engine_options.world_size)
        self.all_gather = all_gather
        self.last_exchange: Dict[str, int] = {}

    def owned(self, indices) -> np.ndarray:
        return block_owner(indices, self.world) == self.rank

    def gather(self) -> Dict[Tuple[int, int, int], np.ndarray]:
        """Every block of the map (all shards), as {index: voxels} on every rank."""
        idx = self.layer.getAllAllocatedBlocks()
        vox, _ = self.layer.getBlocks(idx)
        if len(idx):
            mine = self.owned(idx)
            idx, vox = idx[mine], vox[mine]
        all_idx, all_vox, _ = all_gather_blocks(idx, vox, self.group)
        dt = vox.dtype
        return {tuple(int(v) for v in i): all_vox[k].view(dt) for k, i in enumerate(all_idx)}

    def sync_replicas(self, updated_mask: int = 1) -> int:
        """Make every rank's map a full replica for READING: all-gather the owned blocks dirtied since
        the last call (Update::kMap bit by default, cleared on the owner) and upload the other ranks'
        blocks as read-only copies (the integrators never touch blocks this rank does not own).
        Returns the number of blocks received."""
        idx, vox, _ = self.layer.mirrorUpdated(updated_mask, clear_mask=updated_mask)
        if len(idx):
            mine = self.owned(idx)
            idx, vox = idx[mine], vox[mine]
        all_idx, all_vox, counts = all_gather_blocks(idx, vox, self.group)
        if not len(all_idx):
            return 0
        theirs = ~self.owned(all_idx)
        if theirs.any():
            self.layer.insertBlocks(all_idx[theirs], all_vox[theirs].view(vox.dtype).reshape(int(theirs.sum()), -1),
                                    updated_bits=np.zeros(int(theirs.sum()), np.uint8))
        return int(theirs.sum())

    def exchange(self, layer: Optional[Layer] = None) -> int:
        """Bring every rank's read-only replicas of the other ranks' blocks up to date, GPU to GPU.

        1. The blocks this rank owns that changed since the last exchange (the engine's own
           VBX_UPDATED_MIRROR mark, cleared here; the owner's kMap / kMesh / kEsdf bits stay with its own
           consumers) are gathered on the device into one padded CUDA buffer.
        2. One all-gather of the counts, one all-gather of the indices and payloads.
        3. The other ranks' blocks are written into this rank's map with REPLICA_BITS set.
        Afterwards every rank holds the whole map as of the last scan.  Block removals do not propagate:
        the caller removes a block on every rank.  `layer` defaults to the TSDF shard (an ESDF Layer of the
        same engine may be passed).  Returns the number of blocks received; `last_exchange` holds the
        counts and bytes of the call."""
        import torch

        lay = self.layer if layer is None else layer
        opt = lay.engine_options
        dev = torch.device("cuda", opt.device if opt is not None and opt.device >= 0 else torch.cuda.current_device())
        bb = lay._block_bytes()
        n = lay.gatherUpdatedDevice(UPDATED_MIRROR, owned_only=True)  # the count only (cap 0: nothing cleared)
        counts = torch.zeros(self.world, dtype=torch.int64, device=dev)
        self.all_gather(counts, torch.full((1,), n, dtype=torch.int64, device=dev))
        counts = counts.tolist()
        cap = int(max(counts))
        self.last_exchange = dict(sent=n, received=0, bytes=0)
        if cap == 0:
            return 0
        # one buffer per rank: cap payloads (16-byte aligned for the gather's vector stores), then cap indices
        per = cap * (bb + 12)
        send = torch.empty(per, dtype=torch.uint8, device=dev)
        if lay.gatherUpdatedDevice(UPDATED_MIRROR, clear_mask=UPDATED_MIRROR, owned_only=True,
                                   d_idx3=send[cap * bb:cap * bb + 12 * n], d_voxels=send[:n * bb], cap=n) != n:
            raise VoxbloxError("the owned dirty blocks changed between the count and the gather")
        recv = torch.empty(self.world * per, dtype=torch.uint8, device=dev)
        self.all_gather(recv, send)
        torch.cuda.current_stream(dev).synchronize()  # (the engine reads recv on its own stream)
        got = 0
        for r, c in enumerate(counts):
            if r == self.rank or c == 0:
                continue
            base = r * per
            lay.insertBlocksDevice(recv[base + cap * bb:base + cap * bb + 12 * c], recv[base:base + c * bb], m=c,
                                   updated_bits=REPLICA_BITS)
            got += c
        self.last_exchange = dict(sent=n, received=got, bytes=got * (bb + 12))
        return got
