"""Timing of the action sampler alone: fused megakernel (csrc/dit_sampler.cu) vs the module path, batch 1 and 2.
At batch 2 the FUSED_SAMPLER run is also the module path (two sequences are 24 rows, the kernel takes 12), called eagerly
instead of replayed as a graph: that row measures launch overhead, not the kernel.
   python tools/prof_sampler.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tests import synth  # noqa: E402
from tests.test_rollout_gpu import build  # noqa: E402

dev = torch.device("cuda:0")
model = build(synth.CASES["libero_dit"], dev)
g = torch.Generator().manual_seed(1)
for bs in (1, 2):
    feat = (torch.randn(bs, 3, 1024, generator=g) * 0.7).to(dev, torch.bfloat16)
    noise = torch.randn(bs, 3, 7, generator=g).to(dev)
    for fused in (True, False):
        model.FUSED_SAMPLER = fused
        with torch.no_grad():
            for _ in range(3):
                model._ddim_actions(feat, noise, dev)
            torch.cuda.synchronize()
            if not fused:       # the module path is launch-bound: time it the way the wrapper runs it, as a CUDA graph
                gph = torch.cuda.CUDAGraph()
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    model._ddim_actions(feat, noise, dev)
                torch.cuda.current_stream().wait_stream(side)
                with torch.cuda.graph(gph):
                    model._ddim_actions(feat, noise, dev)
                run = gph.replay
            else:
                run = lambda: model._ddim_actions(feat, noise, dev)   # noqa: E731
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            run()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(10):
                run()
            e1.record()
            torch.cuda.synchronize()
        label = "module path (graph replay)" if not fused else "fused megakernel" if bs == 1 else "module path (eager)"
        print(f"sampler bs={bs} {label}: {e0.elapsed_time(e1) / 10:.3f} ms",
              flush=True)
