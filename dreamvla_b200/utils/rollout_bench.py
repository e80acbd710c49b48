"""Synthetic rollout driver for the action-latency metric (BASELINE.json configs[3]; SURVEY §8d metric 2): N consecutive
`ModelWrapper.step` calls (growing then sliding window, batch 1), each timed host-side around the call with a device
synchronize on both sides -- preprocessing excluded, as in the reference's loop the simulator sits between calls.
`run_batched` drives a batched wrapper the same way over `num_envs` synthetic envs whose episodes start staggered, so that
every batched step mixes window fill levels."""
from __future__ import annotations

import time

import numpy as np
import torch


def synthetic_text(seed=0):
    g = torch.Generator().manual_seed(seed)
    text = torch.zeros(77, dtype=torch.long)
    text[0], text[1:6], text[6] = 49406, torch.randint(1, 49406, (5,), generator=g), 49407
    return text


def percentile_report(lat_ms, skip):
    lat = np.sort(np.asarray(lat_ms[skip:], dtype=np.float64))
    return {"p50": float(np.percentile(lat, 50)), "p99": float(np.percentile(lat, 99)), "mean": float(lat.mean()),
            "min": float(lat[0]), "max": float(lat[-1]), "timed_steps": int(lat.size), "skipped_warmup_steps": int(skip)}


def run_calvin(wrapper, steps, seed=0, episode_len=360):
    """eval_utils_calvin.py:264 call pattern: reset at episode starts, one step per env tick."""
    g = torch.Generator().manual_seed(seed)
    text = synthetic_text(seed)
    lat = []
    for i in range(steps):
        if i % episode_len == 0:
            wrapper.reset()
        img, grip, obs = torch.randn(3, 224, 224, generator=g), torch.randn(3, 224, 224, generator=g), torch.randn(15, generator=g)
        img, grip = img.pin_memory(), grip.pin_memory()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wrapper.step(img, grip, obs, text)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    return lat


def run_libero(wrapper, steps, seed=0, episode_len=600):
    """eval_utils_libero.py:185-196 call pattern (timestep restarts with every episode)."""
    g = torch.Generator().manual_seed(seed)
    text = synthetic_text(seed)
    lat = []
    for i in range(steps):
        if i % episode_len == 0:
            wrapper.reset()
        img, grip = torch.randn(3, 224, 224, generator=g).pin_memory(), torch.randn(3, 224, 224, generator=g).pin_memory()
        pos = torch.randn(3, generator=g).numpy() * 0.3
        quat = torch.randn(4, generator=g).numpy()
        qpos = torch.rand(2, generator=g).numpy() * 0.04
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wrapper.step(img, grip, pos, quat, qpos, text, i % episode_len)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    return lat


def run_batched(wrapper, steps, kind, seed=0, episode_len=360):
    """`steps` batched steps of all wrapper.num_envs envs (BatchedModelWrapper of eval_utils_calvin / eval_utils_libero,
    `kind` "calvin" / "libero"); env e starts its first episode e * episode_len // num_envs steps into its cycle.
    -> per-batched-step latencies in ms."""
    N = wrapper.num_envs
    g = torch.Generator().manual_seed(seed)
    text = synthetic_text(seed).expand(N, 77)
    envs = list(range(N))
    offset = [e * episode_len // N for e in envs]
    lat = []
    for i in range(steps):
        ts = [(i + offset[e]) % episode_len for e in envs]
        for e in envs:
            if ts[e] == 0 or i == 0:
                wrapper.reset(e)
        img, grip = torch.randn(N, 3, 224, 224, generator=g).pin_memory(), torch.randn(N, 3, 224, 224, generator=g).pin_memory()
        if kind == "calvin":
            obs = torch.randn(N, 15, generator=g)
            call = lambda: wrapper.step(envs, img, grip, obs, text)                                    # noqa: E731
        else:
            pos, quat = torch.randn(N, 3, generator=g).numpy() * 0.3, torch.randn(N, 4, generator=g).numpy()
            qpos = torch.rand(N, 2, generator=g).numpy() * 0.04
            call = lambda: wrapper.step(envs, img, grip, pos, quat, qpos, text, ts)                     # noqa: E731
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    return lat


def batched_report(lat, skip, num_envs, mode):
    rep = percentile_report(lat, skip)
    return {**rep, "num_envs": int(num_envs), "mode": mode, "actions_per_s": float(num_envs * 1e3 / rep["p50"])}
