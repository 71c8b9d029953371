"""Data-parallel sharding over images + one all-gather of per-image output records.

The path shards naturally: images are independent (the reference is batch-1 and has no
cross-image op; SURVEY.md section 8e), so there is no collective inside the forward.  One process
per GPU (`torch.distributed`, NCCL over NVLink/NVSwitch; gloo in the CPU tests);
weights are replicated; the only exchange is a single all-gather of fixed-size records:
    [count | boxes 600x4 | scores 600x21 | masks 600x441]  fp32  (~1.12 MB per image).
"""
import os

import torch
import torch.distributed as dist

from .engine import ROIS_PER_IMAGE, MASK_SIZE, NUM_CLASSES

N_DET = 2 * ROIS_PER_IMAGE
MSZ = MASK_SIZE * MASK_SIZE


def record_len(B):
    """Floats in the output record of a B-image step (ops.record_layout): counts[B] (padded to a
    multiple of 4) | boxes[B][600][4] | scores[B][600][21] | masks[B][600][441]."""
    from .ops import record_layout
    return record_layout(B, ROIS_PER_IMAGE, MSZ, NUM_CLASSES)[3]


def init_from_env(backend=None):
    """Reads RANK / WORLD_SIZE / LOCAL_RANK / MASTER_* (torchrun).  Returns (rank, world, local)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, world, local


def shard_range(total, rank, world):
    """Contiguous block partition of `total` images: ranks [0, total % world) get one extra."""
    base, rem = divmod(total, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def pack_records(boxes, masks, scores, valid):
    """(B,600,4), (B,600,1,21,21), (B,600,21), (B,600) -> the record (1-D fp32) in the layout the
    engine's detect tail writes on the device (torch restatement: CPU tests, host-side callers)."""
    from .ops import record_layout
    B = boxes.shape[0]
    ob, os_, om, end = record_layout(B, ROIS_PER_IMAGE, MSZ, NUM_CLASSES)
    rec = torch.zeros(end, dtype=torch.float32, device=boxes.device)
    rec[:B] = valid.view(B, -1).to(torch.float32).sum(dim=1)
    rec[ob:os_] = boxes.reshape(-1)
    rec[os_:om] = scores.reshape(-1)
    rec[om:end] = masks.reshape(-1)
    return rec


def unpack_records(allrec, B):
    """(world, record_len(B)) -> count (world*B,) int64, boxes, masks, scores in global image order
    (rank-major = image order for contiguous shards)."""
    from .ops import record_views
    parts = [record_views(allrec[r], B, ROIS_PER_IMAGE, MSZ, NUM_CLASSES) for r in range(allrec.shape[0])]
    count = torch.cat([p[0] for p in parts]).round().to(torch.int64)
    return (count, torch.cat([p[1] for p in parts]), torch.cat([p[3] for p in parts]),
            torch.cat([p[2] for p in parts]))


def all_gather_records(rec, out=None):
    """Every rank contributes its record and receives (world, len): the one collective of a step.
    Equal per-rank batch (the bench's weak-scaling layout)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return rec.view(1, -1)
    world = dist.get_world_size()
    if out is None:
        out = torch.empty((world, rec.numel()), dtype=rec.dtype, device=rec.device)
    dist.all_gather_into_tensor(out.view(-1), rec)
    return out


class GatherPipe:
    """The step's all-gather on a side stream, double-buffered, so that it overlaps the next
    step's trunk: `submit(rec)` returns at once; the gathered tensor of step k is complete on the
    main stream after `wait(k)` (or `drain()`).  With world 1 it is a no-op."""

    def __init__(self, device, rec_len, depth=2):
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.device = device
        self.depth = depth
        self.k = 0
        if self.world > 1:
            self.stream = torch.cuda.Stream(device=device)
            self.send = [torch.empty(rec_len, dtype=torch.float32, device=device) for _ in range(depth)]
            self.recv = [torch.empty((self.world, rec_len), dtype=torch.float32, device=device)
                         for _ in range(depth)]
            self.done = [None] * depth

    def send_buffer(self):
        """The record buffer the next step should write (engine.detect_tail(rec=...)); waits on the
        main stream for the gather that last read it."""
        if self.world == 1:
            return None
        slot = self.k % self.depth
        if self.done[slot] is not None:
            torch.cuda.current_stream(self.device).wait_event(self.done[slot])
        return self.send[slot]

    def submit(self):
        if self.world == 1:
            self.k += 1
            return None
        slot = self.k % self.depth
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            dist.all_gather_into_tensor(self.recv[slot].view(-1), self.send[slot])
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.done[slot] = ev
        self.k += 1
        return self.recv[slot]

    def drain(self):
        if self.world > 1:
            torch.cuda.current_stream(self.device).wait_stream(self.stream)
