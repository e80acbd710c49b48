#!/usr/bin/env python
"""bench.py -- train-step samples/sec of the DreamVLA hot path (BASELINE.json metric) on N H100s of one node.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--batch B_per_gpu] [--config calvin|libero]
                  [--dump-outputs DIR]

Workload (config.workload): BASELINE.json configs[1] -- CALVIN ABC-D train step, bf16, sequence_length 10, all five
world-knowledge heads (RGB / depth / DINO / SAM / flow) + DiT action head, L = 1290 backbone tokens, per-GPU batch 2
(scripts/CALVIN_ABC_D/DreamVLA/finetune.sh:21), GPT-2 dropouts 0.1 as in the reference's training mode.
A step = forward + 7 losses + backward + gradient all-reduce (N > 1) + global-norm clip + AdamW.
`value` times steps on device-resident synthetic inputs (CUDA events, barrier + synchronize both sides, max over ranks);
`e2e` times the same public API call with pinned-host inputs copied H2D and the loss copied D2H inside the timed region.
`--dump-outputs DIR` writes what the last timed step produced (see dump_outputs) so that two builds can be compared
output for output: model, weights and batch are seeded, so the inputs are identical from run to run.
`--impl reference` times the reference's own algorithm on the host CPU cores (oracle port of the reference modules,
pinned against the unmodified reference by tests/test_oracle_cpu.py) on a bounded sample of the same workload.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "reference_gpu"])
    ap.add_argument("--batch", type=int, default=8, help="per-GPU batch: SURVEY.md C2 measures B=2 (finetune.sh value) and B=8")
    ap.add_argument("--config", default="calvin", choices=["calvin", "libero"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the extra fields of the default line (reference-on-GPU arm, "
                    "script batch size, LIBERO config, action latency); they only run on 1 GPU")
    ap.add_argument("--latency-steps", type=int, default=1000)
    ap.add_argument("--dropout", type=float, default=0.1)
    ap.add_argument("--no-graph", action="store_true", help="launch every kernel from Python instead of replaying CUDA graphs")
    ap.add_argument("--layers", type=int, default=24, help=argparse.SUPPRESS)  # debugging only; bench lines use 24
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's outputs to DIR/<name>.npy (float32)")
    args = ap.parse_args()
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs writes the outputs of this package's train step; it is not available with --impl " + args.impl)
    return args


CONFIGS = {
    # scripts/CALVIN_ABC_D/DreamVLA/finetune.sh + --dino_feat_pred/--trajectory_pred (SURVEY §8d C2)
    "calvin": dict(model=dict(sequence_length=10, num_resampler_query=16, num_obs_token_per_image=9, obs_pred=True,
                              depth_pred=True, trajectory_pred=True, dino_feat_pred=True, sam_feat_pred=True,
                              action_pred_steps=3, transformer_layers=24, hidden_dim=1024, transformer_heads=16,
                              phase="finetune", track_label_patch_size=8, use_dit_head=True, attn_implementation="sdpa"),
                   step=dict(sequence_length=10, future_steps=3, action_pred_steps=3, use_dit_head=True, loss_action=True,
                             loss_image=True, loss_depth=True, loss_dino_feat=True, loss_sam_feat=True, loss_trajectory=True,
                             flow_as_mask=True, learning_rate=1e-3, weight_decay=1e-4),
                   heads=dict(depth=True, dino=True, sam=True, traj=True),
                   tf_per_sample=7.202, name="CALVIN ABC-D train step, bf16, S=10, L=1290, heads RGB+depth+DINO+SAM+flow, DiT-B"),
    # scripts/LIBERO/DreamVLA/finetune_long.sh minus world heads (SURVEY §8d C3)
    "libero": dict(model=dict(sequence_length=7, num_resampler_query=16, num_obs_token_per_image=9, obs_pred=False,
                              depth_pred=False, trajectory_pred=False, dino_feat_pred=False, sam_feat_pred=False,
                              action_pred_steps=3, transformer_layers=24, hidden_dim=1024, transformer_heads=16,
                              phase="finetune", use_dit_head=True, attn_implementation="sdpa", gripper_width=True),
                   step=dict(sequence_length=7, future_steps=3, action_pred_steps=3, use_dit_head=True, loss_action=True,
                             learning_rate=1e-3, weight_decay=1e-4, gripper_width=True),
                   heads=dict(),
                   tf_per_sample=1.280, name="LIBERO train step, bf16, S=7, L=273, world heads off, DiT-B"),
}


# ----------------------------------------------------------------------------------------------------------------------
class ClockSampler(threading.Thread):
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        super().__init__(daemon=True)
        self.gpu_index = gpu_index
        self.samples = []
        self.stop_flag = threading.Event()

    def _nvml_loop(self):
        """NVML (nvidia_ml_py) polled every 20 ms: one nvidia-smi process takes ~0.5 s to answer, which leaves a 1.6 s timed
        region with one or two samples.  Same fields as the nvidia-smi query; any failure falls back to nvidia-smi."""
        import pynvml as N
        N.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = self.gpu_index
        if vis:                                  # NVML enumerates physical devices, CUDA the visible subset
            ids = [v.strip() for v in vis.split(",") if v.strip()]
            if self.gpu_index < len(ids) and ids[self.gpu_index].isdigit():
                idx = int(ids[self.gpu_index])
        h = N.nvmlDeviceGetHandleByIndex(idx)
        mx = N.nvmlDeviceGetMaxClockInfo(h, N.NVML_CLOCK_SM)
        bits = (("hw_slowdown", N.nvmlClocksEventReasonHwSlowdown), ("hw_thermal_slowdown", N.nvmlClocksEventReasonHwThermalSlowdown),
                ("sw_thermal_slowdown", N.nvmlClocksEventReasonSwThermalSlowdown), ("sw_power_cap", N.nvmlClocksEventReasonSwPowerCap))
        while not self.stop_flag.is_set():
            sm = N.nvmlDeviceGetClockInfo(h, N.NVML_CLOCK_SM)
            r = N.nvmlDeviceGetCurrentClocksEventReasons(h)
            pw = N.nvmlDeviceGetPowerUsage(h) / 1000.0
            self.samples.append([str(idx), str(sm), str(mx), f"{pw:.1f}"] + ["Active" if r & b else "Not Active" for _, b in bits])
            self.stop_flag.wait(0.02)

    def run(self):
        try:
            self._nvml_loop()
            return
        except Exception:  # noqa: BLE001   (no NVML binding / driver mismatch: the nvidia-smi recipe)
            pass
        while not self.stop_flag.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i",
                                      str(self.gpu_index)], capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.samples.append([x.strip() for x in out.split(",")])
            except Exception:  # noqa: BLE001
                pass
            self.stop_flag.wait(0.2)

    def summary(self):
        sm, reasons, mx = [], set(), None
        for s in self.samples:
            try:
                sm.append(float(s[1]))
                mx = float(s[2])
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), s[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            except Exception:  # noqa: BLE001
                continue
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


# Dense BF16 tensor-core rate of the H100 SXM from NVIDIA's data sheet (700 W part): the denominator of the "frac" fields,
# not a rate this code has reached.
H100_BF16_DENSE_TFLOPS = 989.0
PEAK_SOURCE = "NVIDIA H100 SXM data sheet, dense BF16 (not measured)"


def dump_outputs(out_dir, loss, params):
    """What a caller of the timed train step receives from its last step: the loss it returns, and the model it updates in
    place -- as a fixed, seeded sample of 4 Mi elements of the flat bf16 parameter buffer (16 MB as float32; the whole buffer
    is ~1.3 GB).  Written as float32 .npy files."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), loss.detach().float().reshape(1).cpu().numpy())
    n = params.numel()
    idx = torch.randint(0, n, (min(n, 4 << 20),), generator=torch.Generator().manual_seed(0)).sort().values
    np.save(os.path.join(out_dir, "params_sample.npy"), params.detach()[idx.to(params.device)].float().cpu().numpy())


# ----------------------------------------------------------------------------------------------------------------------
def build_model(cfg, device, dropout, layers=None):
    from dreamvla_b200.models import DreamVLA
    mk = dict(cfg["model"])
    if layers is not None:
        mk["transformer_layers"] = layers
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **mk)
    model = model.bfloat16().to(device)
    model.clip_model.requires_grad_(False)
    model._init_model_type()
    model.train()
    gp = model.transformer_backbone
    gp.embd_pdrop = dropout
    for blk in gp.h:
        blk.attn.attn_pdrop = blk.attn.resid_pdrop = blk.mlp.resid_pdrop = dropout
    return model


def run_ours(args):
    import torch.distributed as dist
    from dreamvla_b200 import _lib
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, StepConfig, TrainStep, synthetic_batch

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("bench.py --gpus N>1 must be launched with torch.distributed.run (one rank per GPU)")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    verbose = bool(os.environ.get("DVLA_BENCH_VERBOSE"))
    t_begin = time.perf_counter()

    def stage(msg):
        if verbose:
            print(f"[bench r{rank} +{time.perf_counter() - t_begin:6.1f}s] {msg}", file=sys.stderr, flush=True)
    if world > 1:
        from dreamvla_b200.utils.distributed_utils import configure_nccl
        configure_nccl()
        dist.init_process_group("nccl", device_id=dev)
    stage("process group up")
    cfg = CONFIGS[args.config]
    scfg = StepConfig(**cfg["step"])
    model = build_model(cfg, dev, args.dropout, args.layers)
    step = TrainStep(model, scfg, world_size=world)
    if world > 1:   # DDP ctor semantics: rank 0's parameters everywhere
        dist.broadcast(step.flat.P, src=0)
    heads = dict(cfg["heads"], flow_mask=scfg.flow_as_mask)
    B = args.batch
    batch = synthetic_batch(scfg, B, dev, seed=1234 + rank, heads=heads)

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    eager_step = step
    graphed = False
    stage("model + batch built")
    if not args.no_graph:
        try:
            step = GraphedTrainStep(eager_step, batch, warmup=3)
            batch = step.static
            graphed = True
            stage("graphs captured")
        except Exception as e:  # noqa: BLE001  (same kernels either way; only the launch mechanism differs)
            print(f"[bench] CUDA-graph capture failed, launching eagerly: {e!r}", file=sys.stderr, flush=True)
            torch.cuda.synchronize()
            step = eager_step

    # ---- device-resident timing ----
    for _ in range(max(args.warmup, 3)):
        loss = step(batch)
    sync_all()
    stage("warm-up done")
    sampler = ClockSampler(local_rank) if rank == 0 else None
    if sampler:
        sampler.start()
    n0 = _lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync_all()
    cuprof = bool(os.environ.get("DVLA_BENCH_CUPROF"))      # `ncu --profile-from-start off`: profile exactly the timed steps
    if cuprof:
        torch.cuda.cudart().cudaProfilerStart()
    e0.record()
    for _ in range(args.steps):
        loss = step(batch)
    e1.record()
    sync_all()
    if cuprof:
        torch.cuda.cudart().cudaProfilerStop()
    ms = e0.elapsed_time(e1)
    launches = _lib.launch_count() - n0
    if graphed:   # replays do not pass through the host-side counter: kernels recorded per step x replays
        launches = step.launches_per_step * args.steps
    if sampler:
        sampler.stop_flag.set()
        sampler.join()
    t = torch.tensor([ms], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t)
    stage("timed region done")
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, eager_step.flat.P)
    ms_per_step = ms / args.steps
    value = B * world / (ms_per_step / 1e3)
    final_loss = float(loss)

    # ---- end-to-end: pinned host inputs -> H2D -> step -> D2H loss, every step ----
    # measured right after the device-resident loop, in the same power / clock state (the per-shape GEMM microbenchmark of
    # the roofline section keeps the GPU at the power cap for seconds; a region timed after it runs at lower clocks)
    e2e = None
    if not args.no_e2e:
        from dreamvla_b200.utils.train_utils import prefetch_to_device
        host = synthetic_batch(scfg, B, dev, seed=1234 + rank, heads=heads, pin=True)
        loss_host = torch.zeros(1, dtype=torch.float32).pin_memory()
        h2d = sum(v.numel() * v.element_size() for v in host.values())

        def host_batches(n):          # the data loader of this measurement: the same pinned batch, n times
            for _ in range(n):
                yield host

        def e2e_run(n):
            # the public training-loop iterator (train_one_epoch_calvin uses the same one): batch i+1 is copied host->device
            # on a copy stream while step i runs; every step still moves its own 193 MB in and its loss out
            for dbatch in prefetch_to_device(host_batches(n), dev):
                ls = step(dbatch)
                loss_host.copy_(ls.reshape(1).float(), non_blocking=True)
        # diagnostic: one batch's host->device copy alone (idle GPU), on a side stream -- what the overlap has to hide
        cs = torch.cuda.Stream()
        dtmp = {k: torch.empty_like(v, device=dev) for k, v in host.items()}
        c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(cs):
            for k, v in host.items():
                dtmp[k].copy_(v, non_blocking=True)
            c0.record(cs)
            for k, v in host.items():
                dtmp[k].copy_(v, non_blocking=True)
            c1.record(cs)
        torch.cuda.synchronize()
        h2d_alone_ms = c0.elapsed_time(c1)
        del dtmp
        try:
            e2e_run(3)
        except Exception as e:  # noqa: BLE001   (keep the measurement alive: sequential copy -> step -> read-back)
            print(f"[bench] prefetching input pipeline failed ({e!r}); measuring e2e with in-line copies", file=sys.stderr, flush=True)
            dbuf = {k: torch.empty_like(v, device=dev) for k, v in host.items()}

            def e2e_run(n):  # noqa: F811
                for _ in range(n):
                    for k, v in host.items():
                        dbuf[k].copy_(v, non_blocking=True)
                    ls = step(dbuf)
                    loss_host.copy_(ls.reshape(1).float(), non_blocking=True)
            e2e_run(3)
        sync_all()
        sampler2 = ClockSampler(local_rank) if rank == 0 else None
        if sampler2:
            sampler2.start()
        t0 = time.perf_counter()
        e0.record()
        e2e_run(args.steps)
        e1.record()
        sync_all()
        wall = (time.perf_counter() - t0) * 1e3
        if sampler2:
            sampler2.stop_flag.set()
            sampler2.join()
        t = torch.tensor([max(e0.elapsed_time(e1), 0.0)], device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_ms = float(t) / args.steps
        e2e = {"value": round(B * world / (e2e_ms / 1e3), 3), "unit": "samples/s", "h2d_bytes_per_step": h2d,
               "d2h_bytes_per_step": 4, "ms_per_step": round(e2e_ms, 3), "wall_ms_per_step": round(wall / args.steps, 3),
               "h2d_alone_ms": round(h2d_alone_ms, 3), "h2d_alone_gbs": round(h2d / h2d_alone_ms / 1e6, 2),
               "input_pipeline": "train_utils.prefetch_to_device (copy stream, 2 persistent device slots)",
               "clocks": sampler2.summary() if sampler2 else None}

        if os.environ.get("DVLA_E2E_PROBE"):
            # diagnostic (stderr only): which part of the input pipeline costs device time when it runs beside the step
            def timed(fn):
                fn(3)
                sync_all()
                e0.record()
                fn(args.steps)
                e1.record()
                sync_all()
                tt = torch.tensor([e0.elapsed_time(e1) / args.steps], device=dev)
                if world > 1:
                    dist.all_reduce(tt, op=dist.ReduceOp.MAX)
                return float(tt)
            dbf = {k: torch.empty(v.shape, dtype=(torch.bfloat16 if v.is_floating_point() else v.dtype), device=dev) for k, v in host.items()}
            dst = {k: torch.empty_like(v, device=dev) for k, v in host.items()}

            def resident(n):
                for _ in range(n):
                    step(batch)

            def resident_copy_in(n):      # + the device->device copy into the graph's static inputs
                for _ in range(n):
                    step(dbf)

            def dma_beside(n):            # + unsynchronised H2D DMA on a side stream (no cast kernels, no events)
                for _ in range(n):
                    with torch.cuda.stream(cs):
                        for k, v in host.items():
                            dst[k].copy_(v, non_blocking=True)
                    step(batch)

            def dma_cast_beside(n):       # + the fp32 -> bf16 cast kernels on the side stream
                for _ in range(n):
                    with torch.cuda.stream(cs):
                        for k, v in host.items():
                            dst[k].copy_(v, non_blocking=True)
                            if v.is_floating_point():
                                dbf[k].copy_(dst[k])
                    step(batch)

            def prefetch3(n):
                for dbatch in prefetch_to_device(host_batches(n), dev, slots=3):
                    step(dbatch)
            def resident_d2h(n):          # + the loss read-back of every step
                for _ in range(n):
                    ls = step(batch)
                    loss_host.copy_(ls.reshape(1).float(), non_blocking=True)

            def prefetch_no_d2h(n):
                for dbatch in prefetch_to_device(host_batches(n), dev):
                    step(dbatch)
            for name, fn in (("resident", resident), ("resident+d2h_loss", resident_d2h), ("resident+copy_in", resident_copy_in),
                             ("dma_beside", dma_beside), ("dma+cast_beside", dma_cast_beside), ("prefetch(2) no d2h", prefetch_no_d2h),
                             ("prefetch(2)", e2e_run), ("prefetch(3)", prefetch3), ("resident", resident)):
                tms = timed(fn)
                if rank == 0:
                    print(f"[e2e probe] world={world} {name:18s} {tms:8.3f} ms/step", file=sys.stderr, flush=True)

    stage("e2e done")
    # ---- roofline of the dominant kernel (wgmma GEMM) ------------------------------------------------------------------
    # one eager fwd+bwd records every dvla_gemm launch (shape, layout, epilogue); each distinct launch is then re-issued
    # 5x back to back on the current stream between two CUDA events (no host gaps), and
    #   achieved = sum(count * 2MNK) / sum(count * avg duration)
    roof = None
    if rank == 0:
        from collections import Counter
        calls = Counter()
        orig = _lib.gemm

        def rec_gemm(a, b, **kw):
            a_mn, b_mn = kw.get("a_mn", False), kw.get("b_mn", False)
            M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
            N = b.shape[1] if b_mn else b.shape[0]
            tma = a.stride(0) % 8 == 0 and b.stride(0) % 8 == 0
            calls[(M, N, K, a_mn, b_mn, kw.get("bias") is not None, int(kw.get("act", 0)), kw.get("residual") is not None,
                   kw.get("aux_out") is not None, float(kw.get("dropout_p", 0.0)) > 0, tma, kw.get("aux_in") is not None)] += 1
            return orig(a, b, **kw)
        _lib.gemm = rec_gemm
        try:
            eager_step.forward_backward(batch)
        finally:
            _lib.gemm = orig
        torch.cuda.synchronize()
        eager_step.flat.G.zero_()
        fl = tm = 0.0
        n_tc = 0
        for (M, N, K, a_mn, b_mn, hb, act, hr, ha, hd, tma, hai), cnt in calls.items():
            if not tma:
                continue
            A = torch.randn((K, M) if a_mn else (M, K), device=dev, dtype=torch.bfloat16)
            Bm = torch.randn((K, N) if b_mn else (N, K), device=dev, dtype=torch.bfloat16)
            kw = dict(a_mn=a_mn, b_mn=b_mn, act=act, bias=torch.zeros(N, device=dev, dtype=torch.bfloat16) if hb else None,
                      residual=torch.zeros(M, N, device=dev, dtype=torch.bfloat16) if hr else None,
                      aux_out=torch.empty(M, N, device=dev, dtype=torch.bfloat16) if ha else None,
                      aux_in=torch.zeros(M, N, device=dev, dtype=torch.bfloat16) if hai else None,
                      out=torch.empty(M, N, device=dev, dtype=torch.bfloat16), dropout_p=0.1 if hd else 0.0, dropout_seed=1)
            for _ in range(2):
                orig(A, Bm, **kw)
            s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            for _ in range(5):
                orig(A, Bm, **kw)
            s1.record()
            torch.cuda.synchronize()
            per = s0.elapsed_time(s1) / 5
            tm += cnt * per
            fl += cnt * 2.0 * M * N * K
            n_tc += cnt
            if os.environ.get("DVLA_BENCH_DUMP"):
                print(f"[gemm] M={M:6d} N={N:5d} K={K:5d} a_mn={int(a_mn)} b_mn={int(b_mn)} bias={int(hb)} act={act} res={int(hr)} "
                      f"aux={int(ha)} drop={int(hd)} n={cnt:4d} {per*1e3:8.1f} us {2.0*M*N*K/per/1e9:7.0f} TF/s total {cnt*per:7.3f} ms",
                      file=sys.stderr, flush=True)
        peak = H100_BF16_DENSE_TFLOPS
        ach = fl / (tm * 1e-3) / 1e12 if tm > 0 else 0.0
        roof = {"bound": "tensor", "kernel": "gemm_wgmma_kernel (every tensor-core GEMM launch of one fwd+bwd)",
                "achieved": round(ach, 1), "peak": peak, "unit": "TFLOP/s", "frac": round(ach / peak, 4),
                "peak_source": PEAK_SOURCE, "launches": n_tc, "distinct_launch_shapes": len(calls),
                "gemm_ms_per_step": round(tm, 3), "gemm_share_of_step": round(tm / ms_per_step, 3),
                "gemm_tflop_per_step": round(fl / 1e12, 3),
                "step_model_tflops": round(cfg["tf_per_sample"] * B / (ms_per_step * 1e-3), 1),
                "step_frac_of_peak": round(cfg["tf_per_sample"] * B / (ms_per_step * 1e-3) / peak, 4)}

    stage("roofline done")
    cpu = None
    if rank == 0 and not args.no_cpu_baseline and world == 1:
        cpu = cpu_baseline(args, steps=1, warm=0)

    extras = None
    if rank == 0 and world == 1 and not args.no_extras:
        # free the headline model first: the extra measurements build their own
        workload_params = eager_step.flat.num_params
        step = eager_step = model = batch = None
        import gc
        gc.collect()
        torch.cuda.empty_cache()
        extras = {}
        for key, fn in (("reference_gpu", lambda: reference_gpu_measure(args.config, B, dev)),
                        ("calvin_script_batch", lambda: quick_train_measure("calvin", 2, dev, args.dropout)),
                        ("libero", lambda: quick_train_measure("libero", 16, dev, args.dropout)),
                        ("action_latency", lambda: latency_measure(dev, args.latency_steps))):
            if key == "calvin_script_batch" and (args.config != "calvin" or B == 2):
                continue
            if key == "libero" and args.config == "libero":
                continue
            try:
                t0 = time.perf_counter()
                extras[key] = fn()
                extras[key]["measure_wall_s"] = round(time.perf_counter() - t0, 1)
            except Exception as e:  # noqa: BLE001   (an extra field must never cost the headline line)
                extras[key] = {"error": repr(e)[:300]}
            stage(f"extra {key} done")
        if "value" in extras.get("reference_gpu", {}):
            extras["vs_reference_gpu"] = round(value / extras["reference_gpu"]["value"], 3)
    else:
        workload_params = eager_step.flat.num_params

    if rank == 0:
        line = {
            "metric": "train_step_samples_per_sec", "value": round(value, 3), "unit": "samples/s", "n_gpus": world,
            "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": round(ms_per_step, 3),
            "gpu": torch.cuda.get_device_name(dev), "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": cfg["name"], "per_gpu_batch": B, "global_batch": B * world,
                       "seq_len": cfg["model"]["sequence_length"], "parallelism": f"dp{world}",
                       "dropout": args.dropout, "layers": args.layers, "cuda_graph": graphed,
                       "l2": "inputs+weights+activations per step >> 50 MB L2 (1.3 GB of bf16 weights re-read every step); no explicit flush",
                       "trainable_params": workload_params, "final_loss": final_loss},
            "clocks": sampler.summary() if sampler else None,
            "e2e": e2e, "gpu_launches": int(launches), "roofline": roof, "cpu_baseline": cpu, "extras": extras,
        }
        print(json.dumps(line), flush=True)
    if world > 1:
        # tear-down: CUDA graphs that recorded NCCL kernels must die before the communicator
        step = eager_step = None
        from dreamvla_b200.utils.distributed_utils import shutdown_distributed
        shutdown_distributed()



# ----------------------------------------------------------------------------------------------------------------------
# extra fields of the default line (1 GPU): other SURVEY §8d configurations, so that they are driver-visible
# ----------------------------------------------------------------------------------------------------------------------
def quick_train_measure(config, B, dev, dropout=0.1, steps=10, warmup=3):
    """samples/s of one more (config, per-GPU batch) with the same code path as the headline (CUDA-graph replay, device-
    resident synthetic inputs, CUDA events)."""
    from dreamvla_b200.utils.train_utils import GraphedTrainStep, StepConfig, TrainStep, synthetic_batch
    cfg = CONFIGS[config]
    scfg = StepConfig(**cfg["step"])
    model = build_model(cfg, dev, dropout)
    eager = TrainStep(model, scfg)
    batch = synthetic_batch(scfg, B, dev, seed=99, heads=dict(cfg["heads"], flow_mask=scfg.flow_as_mask))
    step = GraphedTrainStep(eager, batch, warmup=3)
    for _ in range(warmup):
        step(step.static)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step(step.static)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    peak = H100_BF16_DENSE_TFLOPS
    out = {"workload": cfg["name"], "per_gpu_batch": B, "ms_per_step": round(ms, 3), "value": round(B / ms * 1e3, 2),
           "unit": "samples/s", "steps": steps, "step_frac_of_peak": round(cfg["tf_per_sample"] * B / (ms * 1e-3) / peak, 4),
           "final_loss": float(loss)}
    del step, eager, model, batch
    torch.cuda.empty_cache()
    return out


LATENCY_MODEL = dict(sequence_length=10, num_resampler_query=16, num_obs_token_per_image=9, obs_pred=True, depth_pred=True,
                     sam_feat_pred=True, action_pred_steps=3, transformer_layers=24, hidden_dim=1024, transformer_heads=16,
                     phase="evaluate", use_dit_head=True, attn_implementation="sdpa")     # scripts/CALVIN_ABC_D/DreamVLA/eval.sh


def latency_measure(dev, steps):
    """BASELINE.json configs[3] (SURVEY C4): `steps` consecutive ModelWrapper.step calls, batch 1, growing then sliding window,
    p50 / p99 of the host-side wall time around each call (device synchronised on both sides)."""
    from dreamvla_b200.models import DreamVLA
    from dreamvla_b200.utils import rollout_bench
    from dreamvla_b200.utils.eval_utils_calvin import ModelWrapper
    torch.manual_seed(0)
    model = DreamVLA(finetune_type="calvin", clip_device="cpu", vit_checkpoint_path=None, **LATENCY_MODEL).bfloat16().to(dev)
    model._init_model_type()
    model.eval()
    out = {"workload": "eval_calvin.py action inference (eval.sh heads obs+depth+sam, DiT, S=10, L=930), batch 1", "steps": steps}
    for name, kw in (("full_window", dict(incremental=False)), ("incremental", dict(incremental=True, prune=True))):
        w = ModelWrapper(model, history_len=10, action_pred_steps=3, device=dev, **kw)
        lat = rollout_bench.run_calvin(w, steps, seed=1)
        out[name] = rollout_bench.percentile_report(lat, skip=25)
        del w
        torch.cuda.empty_cache()
    out["unit"] = "ms"
    del model
    torch.cuda.empty_cache()
    return out


# ----------------------------------------------------------------------------------------------------------------------
# the reference's algorithm on the GPU, the way the reference runs it: torch eager kernels + cuBLAS + SDPA with the dense
# additive mask, bf16 (`--precision bf16` casts the model, train.py:122-123), DistributedDataParallel(find_unused_parameters
# =True) (train.py:173), clip_grad_norm_(0.1) + torch.optim.AdamW every step (train_utils.py:599-608).  The modules are the
# oracle's functional restatement (pinned to the unmodified reference by tests/test_oracle_cpu.py), so that this arm needs
# nothing outside the repository.
# ----------------------------------------------------------------------------------------------------------------------
def reference_gpu_measure(config, B, dev, steps=5, warmup=3, world=1):
    import torch.nn.functional as F
    from oracle import dreamvla_oracle as O
    from tests import synth
    from tests.state_template import build_template
    cfg = CONFIGS[config]
    mk = dict(cfg["model"], batch=B, weight_seed=1, input_seed=2 + int(os.environ.get("RANK", "0")))
    sd = {k: (v.to(dev, torch.bfloat16) if v.is_floating_point() else v.to(dev))
          for k, v in synth.synth_state_dict(build_template(mk), 1).items()}
    frozen = ("vision_encoder.", "clip_model.", "attention_mask", "position_embedding")
    names = [k for k, v in sd.items() if v.is_floating_point() and not any(f in k for f in frozen)]
    inp = {k: (v.to(dev, torch.bfloat16) if v.is_floating_point() else v.to(dev)) for k, v in synth.synth_inputs(mk).items()}
    lab = {k: v.to(dev, torch.bfloat16) for k, v in synth.synth_labels(mk).items()} if cfg["heads"] else {}
    S = mk["sequence_length"]
    n = 8 * B * S
    lcfg = dict(mk, future_steps=3, flow_as_mask=cfg["step"].get("flow_as_mask", False))

    def mha_sdpa(q, k, v, scale, mask=None):        # GPT2SdpaAttention / timm fused attention (gpt2.py:196-284)
        q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))
        if mask is not None:                        # dense additive [B, 1, L, L] mask, as dreamvla_model.py:769-775 builds it
            mask = mask.to(q.dtype).expand(q.shape[0], 1, -1, -1).contiguous() if mask.dim() == 2 else mask.to(q.dtype)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=scale).permute(0, 2, 1, 3)
        return o.reshape(o.shape[0], o.shape[1], -1)

    class RefModule(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.params = torch.nn.ParameterList([torch.nn.Parameter(sd[k]) for k in names])

        def forward(self, noise, tstep, drop):
            full = dict(sd)
            full.update(zip(names, self.params))
            with torch.autocast("cuda", dtype=torch.bfloat16):
                fwd = O.dreamvla_forward(full, mk, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                         action_label=inp["action_label"], diffusion_noise=noise, diffusion_timestep=tstep,
                                         diffusion_drop_ids=drop)
                return O.train_losses(lcfg, fwd, lab)["loss"] if cfg["heads"] else fwd["loss_action"]
    mod = RefModule().to(dev)
    run_mod = mod
    if world > 1:
        from torch.nn.parallel import DistributedDataParallel as DDP
        run_mod = DDP(mod, device_ids=[dev.index], find_unused_parameters=True)
    opt = torch.optim.AdamW(mod.parameters(), lr=1e-3, weight_decay=1e-4)
    orig = O._mha
    O._mha = mha_sdpa
    try:
        def one():
            noise = torch.randn(n, 3, 7, device=dev, dtype=torch.bfloat16)
            tstep = torch.randint(0, 100, (n,), device=dev)
            drop = torch.rand(n, device=dev) < 0.1
            loss = run_mod(noise, tstep, drop)
            loss.float().backward()
            torch.nn.utils.clip_grad_norm_(mod.parameters(), 0.1)
            opt.step()
            opt.zero_grad()
            return loss
        for _ in range(warmup):
            one()
        torch.cuda.synchronize()
        if world > 1:
            torch.distributed.barrier()
            torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = one()
        e1.record()
        torch.cuda.synchronize()
        if world > 1:
            torch.distributed.barrier()
        ms = e0.elapsed_time(e1) / steps
        if world > 1:
            t = torch.tensor([ms], device=dev)
            torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
            ms = float(t)
    finally:
        O._mha = orig
    out = {"impl": "reference algorithm on this GPU: torch eager + cuBLAS + SDPA (dense mask), bf16 weights + autocast, "
                   "clip_grad_norm_ + torch.optim.AdamW" + (", DDP find_unused_parameters" if world > 1 else ""),
           "workload": cfg["name"], "per_gpu_batch": B, "ms_per_step": round(ms, 2), "value": round(B * world / ms * 1e3, 2),
           "unit": "samples/s", "steps": steps, "loss": float(loss)}
    del mod, run_mod, opt, sd
    torch.cuda.empty_cache()
    return out


def run_reference_gpu(args):
    import torch.distributed as dist
    rank, local_rank, world = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("LOCAL_RANK", "0"), ("WORLD_SIZE", "1")))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    r = reference_gpu_measure(args.config, args.batch, dev, steps=args.steps, warmup=max(args.warmup, 3), world=world)
    if rank == 0:
        cfg = CONFIGS[args.config]
        print(json.dumps({"impl": "reference_gpu", "metric": "train_step_samples_per_sec", "value": r["value"], "unit": "samples/s",
                          "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": r["ms_per_step"],
                          "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                          "config": {"workload": cfg["name"], "per_gpu_batch": args.batch, "global_batch": args.batch * world,
                                     "seq_len": cfg["model"]["sequence_length"], "parallelism": f"dp{world}"},
                          "how": r["impl"]}), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


# ----------------------------------------------------------------------------------------------------------------------
def usable_cores(cap=32):
    """Host threads actually available to this process: affinity mask and cgroup CPU quota, capped (OpenMP scaling of
    the many small fp32 ops of this workload collapses beyond a few dozen threads)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(int(q) / int(per))))
    except Exception:  # noqa: BLE001
        pass
    return max(1, min(n, cap))


def cpu_baseline(args, steps=1, warm=0, budget_s=150.0):
    """The reference's algorithm (oracle port, fp32) on the host cores: fwd + losses + bwd + clip + AdamW, B = 1 window."""
    from oracle import dreamvla_oracle as O
    from tests import synth
    from tests.state_template import build_template
    cfg = CONFIGS[args.config]
    mk = dict(cfg["model"], batch=1, weight_seed=1, input_seed=2)
    if args.layers is not None:
        mk["transformer_layers"] = args.layers
    cores = usable_cores()
    torch.set_num_threads(cores)
    sd = synth.synth_state_dict(build_template(mk), 1)
    frozen = ("vision_encoder.", "clip_model.", "attention_mask", "position_embedding")
    params = []
    for k, v in sd.items():
        if v.is_floating_point() and not any(f in k for f in frozen):
            v.requires_grad_(True)
            params.append(v)
    opt = torch.optim.AdamW(params, lr=1e-3, weight_decay=1e-4)
    inp = synth.synth_inputs(mk)
    S = mk["sequence_length"]
    lab = synth.synth_labels(mk)
    g = torch.Generator().manual_seed(3)
    noise = torch.randn(8 * S, 3, 7, generator=g)
    tstep = torch.randint(0, 100, (8 * S,), generator=g)
    drop = torch.rand(8 * S, generator=g) < 0.1
    lcfg = dict(mk, future_steps=3, flow_as_mask=cfg["step"].get("flow_as_mask", False))

    def one():
        opt.zero_grad(set_to_none=True)
        with torch.no_grad():   # the reference runs ViT and CLIP under no_grad (dreamvla_model.py:643,670)
            pass
        fwd = O.dreamvla_forward(sd, mk, inp["image_primary"], inp["image_wrist"], inp["state"], inp["text_token"],
                                 action_label=inp["action_label"], diffusion_noise=noise, diffusion_timestep=tstep,
                                 diffusion_drop_ids=drop)
        losses = O.train_losses(lcfg, fwd, lab)
        losses["loss"].backward()
        torch.nn.utils.clip_grad_norm_(params, 0.1)
        opt.step()
        return float(losses["loss"].detach())
    times = []
    t_all = time.perf_counter()
    for i in range(warm + steps):
        t0 = time.perf_counter()
        one()
        dt = time.perf_counter() - t0
        if i >= warm:
            times.append(dt)
        if budget_s is not None and time.perf_counter() - t_all > budget_s and len(times) >= 1:
            break
    sec = sum(times) / len(times)
    return {"value": round(1.0 / sec, 5), "unit": "samples/s", "cores": cores, "kind": "port",
            "sample": f"{len(times)} train step(s) (fwd+7 losses+bwd+clip+AdamW, fp32) of ONE sample window (B=1) of the same "
                      f"workload; {sec:.1f} s/step", "steps_timed": len(times), "s_per_step": round(sec, 2)}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cfg = CONFIGS[args.config]
    cb = cpu_baseline(args, steps=args.steps, warm=min(args.warmup, 1), budget_s=None)   # --steps timed steps, however long
    line = {"impl": "reference", "metric": "train_step_samples_per_sec", "value": cb["value"], "unit": "samples/s",
            "n_gpus": args.gpus, "steps": cb["steps_timed"], "warmup": min(args.warmup, 1),
            "ms_per_step": round(cb["s_per_step"] * 1e3, 1), "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": cfg["name"], "per_gpu_batch": 1, "global_batch": 1,
                       "seq_len": cfg["model"]["sequence_length"], "parallelism": "cpu"},
            "cpu_baseline": cb,
            "e2e": {"value": cb["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    elif a.impl == "reference_gpu":
        run_reference_gpu(a)
    else:
        run_ours(a)
