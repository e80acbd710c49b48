"""The flow-matching (`--use_fm`) integrator of the fused sampler without a GPU: the C ABI refuses what the kernel does not
implement (integrators, step counts, batches other than one sequence) on the host, before any launch, and the host's
timestep inputs are the module path's fp32 values bit for bit."""
import ctypes
import struct

import pytest
import torch

DVLA_ERR_INVALID, DVLA_ERR_UNSUPPORTED = -1, -3


def _args(integrator, n_steps=10, t_values=True, batch=1):
    """A DiT-B-shaped dvla_dit_sampler_args whose device pointers are never dereferenced: every call below is refused by the
    host-side checks."""
    from dreamvla_b200 import _lib as L
    depth, hidden, heads = 2, 768, 12
    blocks = (L.DitBlockWeights * depth)(*[L.DitBlockWeights(*[4096 * (i + 1)] * 8) for i in range(depth)])
    a = L.DitSamplerArgs()
    for n, t in L.DitSamplerArgs._fields_:
        if t is L._vp:
            setattr(a, n, 8192)
    a.blocks = blocks
    a.depth, a.hidden, a.heads, a.mlp, a.token, a.freq, a.channels, a.T, a.batch = depth, hidden, heads, 4 * hidden, 1024, 256, 7, 3, batch
    a.n_steps, a.cfg_scale, a.workspace_bytes = n_steps, 1.0, 1 << 30
    a.integrator = integrator
    if t_values:
        a.t_values = (L._f32 * n_steps)(*L.fm_t_values(n_steps))
    return a


@pytest.mark.parametrize("case", ["integrator_2", "integrator_-1", "fm_null_t_values", "fm_13_steps", "ddim_13_steps",
                                  "batch_2", "batch_0"])
def test_fused_sampler_refuses_on_host(case):
    from dreamvla_b200 import _lib as L
    lib = L.load()
    a, want, text = {
        "integrator_2": (_args(2), DVLA_ERR_UNSUPPORTED, "integrator 2 unsupported (0 DDIM, 1 flow-matching Euler)"),
        "integrator_-1": (_args(-1), DVLA_ERR_UNSUPPORTED, "integrator -1 unsupported (0 DDIM, 1 flow-matching Euler)"),
        "fm_null_t_values": (_args(L.DIT_FM_EULER, t_values=False), DVLA_ERR_INVALID, "needs t_values"),
        "fm_13_steps": (_args(L.DIT_FM_EULER, n_steps=13), DVLA_ERR_UNSUPPORTED, "n_steps 13 above the 12 prologue rows"),
        "ddim_13_steps": (_args(L.DIT_DDIM, n_steps=13, t_values=False), DVLA_ERR_UNSUPPORTED,
                          "n_steps 13 above the 12 prologue rows"),
        "batch_2": (_args(L.DIT_DDIM, t_values=False, batch=2), DVLA_ERR_UNSUPPORTED,
                    "batch 2 unsupported: the fused sampler samples one sequence (batch 1)"),
        "batch_0": (_args(L.DIT_DDIM, t_values=False, batch=0), DVLA_ERR_UNSUPPORTED,
                    "batch 0 unsupported: the fused sampler samples one sequence (batch 1)"),
    }[case]
    n0 = lib.dvla_launch_count()
    rc = lib.dvla_dit_ddim_sample(ctypes.byref(a), None)
    msg = lib.dvla_last_error().decode()
    assert rc == want and text in msg, (case, rc, msg)
    assert lib.dvla_launch_count() == n0


def _bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def test_t_values_are_the_module_paths_fp32_division():
    """FMDiffusion.ddim_sample_loop feeds the DiT `torch.full((n,), float(i)) / T` (gaussian_diffusion.py:169)."""
    from dreamvla_b200 import _lib as L
    got = L.fm_t_values(10)
    assert len(got) == 10
    for i, v in enumerate(got):
        want = (torch.full((1,), float(i)) / 10).item()
        assert _bits(v) == _bits(want), (i, v, want)
    # and through the ctypes array the library reads
    arr = (L._f32 * 10)(*got)
    assert [_bits(arr[i]) for i in range(10)] == [_bits((torch.full((1,), float(i)) / 10).item()) for i in range(10)]
