"""Multi-GPU plumbing: one process per GPU (torchrun), torch.distributed carries the 128-byte NCCL unique id from rank 0
to the other ranks; everything on the data path is NCCL inside libgpx (gpx_dist.cu). The reference has no
multi-device exact-GP path (SURVEY.md §2c/§8e) — block rows of the factor workspace are dealt block-cyclically."""
import ctypes
import os

import numpy as np

from . import _ffi


def block_owner(R, G):
    """rank that owns block row / column block R."""
    return R % G


def chunk_position(R, G, npr):
    """position of block row R's NB x NB chunk in the all-gather panel buffer: chunks are grouped by owner so that each
    rank's contribution is contiguous (gpx_dist.cu: pos = (R mod G) * npr + R div G)."""
    return (R % G) * npr + R // G


def local_slot(R, G):
    """memory-distributed layout (gpx_dist.cu): a rank stores only what it owns; its block row R (R mod G == rank) is its
    local block row R div G of the row-owned workspace, and column block R of U = L^-T its local column block R div G."""
    return R // G


def block_layout(N, NB, G):
    """(Npad, nblk, npr): the matrix is padded to whole NB-blocks, npr = chunks per rank."""
    Npad = -(-N // NB) * NB
    nblk = Npad // NB
    return Npad, nblk, -(-nblk // G)


def shard_rows(N, rank, G):
    """contiguous row shard of rank `rank` for the row-sharded sparse model (the first N mod G ranks get one more row)."""
    base, extra = divmod(N, G)
    lo = rank * base + min(rank, extra)
    return slice(lo, lo + base + (1 if rank < extra else 0))


def exchange_unique_id(make_id, group=None):
    """rank 0 calls make_id() -> 128 bytes; everybody gets them (works on gloo and nccl process groups)."""
    import torch
    import torch.distributed as dist
    rank = dist.get_rank(group)
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    buf = torch.zeros(128, dtype=torch.uint8, device=dev)
    if rank == 0:
        raw = make_id()
        assert len(raw) == 128
        buf.copy_(torch.frombuffer(bytearray(raw), dtype=torch.uint8))
    dist.broadcast(buf, src=0, group=group)
    return bytes(buf.cpu().numpy().tobytes())


def nccl_unique_id():
    raw = ctypes.create_string_buffer(128)
    _ffi.check(_ffi.lib().gpx_comm_unique_id(raw), "gpx_comm_unique_id")
    return raw.raw


def init_engine_comm(engine, group=None):
    """Attach `engine` (one per process, on this process's GPU) to a NCCL communicator spanning the process group."""
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    uid = exchange_unique_id(nccl_unique_id, group)
    _ffi.check(_ffi.lib().gpx_comm_init(engine._h, uid, rank, world), "gpx_comm_init")
    engine.sharded = True   # the joint posterior (single-GPU on the device) takes the reference's host route
    engine.rank, engine.world = rank, world
    return engine
