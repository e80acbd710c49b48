"""Rank discovery and process-group setup -- mirror of reference utils/distributed_utils.py:25-47,103-161 (env-var based,
one process per GPU, NCCL).  Rendezvous defaults to 127.0.0.1."""
from __future__ import annotations

import datetime
import os

import torch


def world_info_from_env():
    local_rank = 0
    for v in ("LOCAL_RANK", "MPI_LOCALRANKID", "SLURM_LOCALID", "OMPI_COMM_WORLD_LOCAL_RANK"):
        if v in os.environ:
            local_rank = int(os.environ[v])
            break
    global_rank = 0
    for v in ("RANK", "PMI_RANK", "SLURM_PROCID", "OMPI_COMM_WORLD_RANK"):
        if v in os.environ:
            global_rank = int(os.environ[v])
            break
    world_size = 1
    for v in ("WORLD_SIZE", "PMI_SIZE", "SLURM_NTASKS", "OMPI_COMM_WORLD_SIZE"):
        if v in os.environ:
            world_size = int(os.environ[v])
            break
    return local_rank, global_rank, world_size


def nccl_cta_budget() -> int:
    """CTAs (= SMs) the gradient all-reduce may occupy while it overlaps the backward pass (DVLA_NCCL_CTAS, default 16)."""
    return max(1, int(os.environ.get("DVLA_NCCL_CTAS", "16")))


def configure_nccl() -> None:
    """Call BEFORE the process group is created.  The all-reduce of the gradient segments runs concurrently with backward's
    persistent GEMMs (one CTA per SM): cap NCCL's CTAs so that the GEMMs can be launched on the remaining SMs
    (TrainStep lowers the kernels' SM budget by the same number while segments are in flight).  NVSwitch / NVLS keeps the
    bus bandwidth of an 8-GPU all-reduce high with few CTAs; an explicit NCCL_MAX_CTAS in the environment wins."""
    os.environ.setdefault("NCCL_MAX_CTAS", str(nccl_cta_budget()))


def init_distributed_device(args):
    args.distributed = False
    if not hasattr(args, "world_size"):
        args.local_rank, args.rank, args.world_size = world_info_from_env()
    if not torch.cuda.is_available():
        raise RuntimeError("dreamvla_b200 needs a CUDA device (H100); there is no CPU path")
    device = torch.device("cuda", args.local_rank)
    torch.cuda.set_device(device)
    if args.world_size > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        configure_nccl()
        torch.distributed.init_process_group(backend=getattr(args, "dist_backend", "nccl"), device_id=device,
                                             timeout=datetime.timedelta(seconds=7200))
        args.distributed = True
    args.device = device
    return device


def shutdown_distributed(timeout_s: float = 20.0):
    """Orderly tear-down for one-process-per-GPU runs.  CUDA graphs that recorded NCCL kernels must be released before the
    communicator: drop every reference to them before calling this.  destroy_process_group() is given `timeout_s`; if it
    does not return (graphs still alive somewhere) the process leaves without it instead of hanging until the launcher's
    timeout."""
    import gc
    import sys
    import threading
    dist = torch.distributed
    if not (dist.is_available() and dist.is_initialized()):
        return
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    dist.barrier()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    sys.stdout.flush()
    th = threading.Thread(target=dist.destroy_process_group, daemon=True)
    th.start()
    th.join(timeout=timeout_s)
    if th.is_alive():
        sys.stderr.flush()
        os._exit(0)
