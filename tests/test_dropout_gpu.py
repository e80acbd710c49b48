"""Dropout on the GPU, checked against the host restatement of the library's Philox masks (tests/philox_ref.py).

Every dropout mask the kernels draw is fully determined by (seed + device counter, element index), so it is compared
bit for bit with the restated mask; the kernels' arithmetic is then compared with plain fp32 references evaluated under
that same mask -- the configuration every training run uses (GPT-2 dropout 0.1), which the model tests cannot reach
because they compare against an oracle with torch's RNG and therefore set every dropout rate to zero.

  * dvla_dropout: y == bf16(x * scale) where kept, 0 where dropped, on the vectorised and the scalar branch, strided and
    in place, for every rounding of (thresh, scale) and seeds / counters that wrap past 2^64.
  * GEMM epilogue: the mask extracted exactly on every path that can carry dropout (wgmma main loop, K-split tail, both
    SIMT kernels, N % 8 != 0), then bias + act + dropout + residual against fp32.
  * attention: the masks of the forward kernel and of the dK/dV backward kernel extracted exactly (q = 0 makes P uniform
    over the visible keys; a one-hot V or dO window then exposes one key or query per output column), on every
    forward/backward kernel pairing, masked and strided forms; the dQ kernel's mask through per-row numeric bars.
  * a CUDA graph of all three, replayed with the device seed counter advanced between replays.
  * a 2-layer GPT-2 backbone in train mode with every dropout at 0.1 against a test-local fp32 forward with the restated
    masks injected: output, input gradient and every parameter gradient.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import philox_ref as R

pytestmark = pytest.mark.gpu

SEED = 0xC0FFEE1234567890            # high 32 bits non-zero: the key's second word matters
WRAP = 2 ** 64 - 5                   # SEED + WRAP wraps past 2^64
SCALE = 0.125                        # 1 / sqrt(64)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def L(dev):
    from dreamvla_b200 import _lib
    _lib.load()
    return _lib


def counter(value, dev):
    """The device seed counter (int64 storage of a uint64) holding `value` mod 2^64."""
    v = int(value) % 2 ** 64
    return torch.tensor([v - 2 ** 64 if v >= 2 ** 63 else v], dtype=torch.int64, device=dev)


def assert_mask(got, want, what, axes):
    got, want = np.asarray(got, dtype=bool), np.asarray(want, dtype=bool)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got != want)
    if len(bad):
        ex = "; ".join(f"{dict(zip(axes, (int(x) for x in idx)))} kernel={'keep' if got[tuple(idx)] else 'drop'}"
                       for idx in bad[:6])
        raise AssertionError(f"{what}: {len(bad)} of {got.size} mask bits differ from the restated Philox mask, e.g. {ex}")


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def row_err(got, ref):
    """Worst relative error over the rows of the last dim (a floor of 0.1 x the RMS row norm keeps near-zero rows from
    dividing by ~0), so that one wrong row or tile fails even when the whole-tensor error is diluted."""
    d = (got.float() - ref.float()).reshape(-1, ref.shape[-1]).norm(dim=1)
    r = ref.float().reshape(-1, ref.shape[-1]).norm(dim=1)
    floor = 0.1 * float(r.pow(2).mean().sqrt()) + 1e-30
    return float((d / r.clamp_min(floor)).max())


# ============================================== dvla_dropout ==========================================================
DROPOUT_CASES = [  # (id, rows, N, ldx, ldy, in_place, p, seed, counter or None)
    ("vec", 37, 1024, 1024, 1024, False, 0.1, SEED, WRAP),
    ("scalar_N1001", 37, 1001, 1001, 1001, False, 0.1, SEED, WRAP),
    ("scalar_N13", 37, 13, 13, 13, False, 0.5, SEED, None),
    ("scalar_N7_seed_wraps", 41, 7, 7, 7, False, 0.9, 2 ** 64 - 1, 3),
    ("vec_ldx", 64, 1024, 1040, 1024, False, 0.1, SEED, 12345),
    ("vec_ldy", 64, 1024, 1024, 1040, False, 0.1, SEED, 12345),
    ("scalar_ldx_odd_ldy", 64, 1001, 1003, 1016, False, 0.1, SEED, 7),
    ("vec_in_place", 64, 1024, 1024, 1024, True, 0.1, SEED, WRAP),
    ("scalar_in_place", 64, 1001, 1001, 1001, True, 0.1, SEED, WRAP),
    ("p_1e-6_keeps_all", 16, 1024, 1024, 1024, False, 1e-6, SEED, WRAP),
    ("p_0.99999", 64, 1024, 1024, 1024, False, 0.99999, SEED, WRAP),
    ("p_0.5_zero_seed_zero_counter", 16, 1024, 1024, 1024, False, 0.5, 0, 0),
]


@pytest.mark.parametrize("case", DROPOUT_CASES, ids=[c[0] for c in DROPOUT_CASES])
def test_dropout_kernel_exact(dev, L, case):
    _, rows, N, ldx, ldy, in_place, p, seed, ctr = case
    g = torch.Generator(device="cpu").manual_seed(rows * N)
    xbuf = (torch.randn(rows, ldx, generator=g) + 0.01).to(dev, torch.bfloat16)
    x = xbuf[:, :N]
    x0 = x.clone()
    if in_place:
        ybuf, y = xbuf, x
    else:
        ybuf = torch.full((rows, ldy), 7.0, device=dev, dtype=torch.bfloat16)
        y = ybuf[:, :N]
    sp = counter(ctr, dev) if ctr is not None else None
    L.dropout(x, p, seed, out=y, seed_ptr=sp)
    torch.cuda.synchronize()
    keep = R.keep_rows(seed, rows, N, p, counter=ctr or 0)
    _, scale = R.thresh_scale(p)
    assert_mask((y != 0).cpu().numpy(), keep, f"dvla_dropout {case[0]}", ("row", "col"))
    want = torch.where(torch.from_numpy(keep).to(dev), (x0.float() * scale).to(torch.bfloat16), torch.zeros_like(x0))
    assert torch.equal(y.view(torch.int16), want.view(torch.int16)), "kept values must be bf16(x * scale) exactly"
    if not in_place and ldy > N:
        assert bool((ybuf[:, N:] == 7.0).all()), "dvla_dropout wrote past N"


# ============================================== GEMM epilogue =========================================================
GEMM_CASES = [  # (id, M, N, K, lda or None, expected kernel, expect a K-split tail)
    ("wgmma", 300, 520, 256, None, 2, False),
    ("wgmma_ksplit_tail", 2580, 1024, 4096, None, 2, True),
    ("wgmma_N1001", 300, 1001, 256, None, 2, False),
    ("wgmma_N7", 960, 7, 768, None, 2, False),
    ("simt_thread", 37, 13, 5, None, 0, False),
    ("simt_warp_lda771", 960, 7, 768, 771, 1, False),
]


def _operands(dev, M, N, K, lda, g, positive):
    abuf = torch.randn(M, lda or K, generator=g)
    w = torch.randn(N, K, generator=g)
    if positive:                       # every pre-dropout value > 0: out == 0 exactly where dropped
        abuf, w = abuf.abs() + 0.05, w.abs() + 0.05
    else:
        abuf, w = abuf * 0.5, w * (0.8 / math.sqrt(K))
    a = abuf.to(dev, torch.bfloat16)[:, :K]
    return a, w.to(dev, torch.bfloat16)


@pytest.mark.parametrize("case", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_dropout_epilogue(dev, L, case):
    name, M, N, K, lda, kernel, tail = case
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    p, ctr = 0.1, WRAP
    sp = counter(ctr, dev)
    keep = R.keep_rows(SEED, M, N, p, counter=ctr)
    _, dscale = R.thresh_scale(p)
    # 1. the mask alone: positive operands, no bias / act / residual
    a, w = _operands(dev, M, N, K, lda, g, positive=True)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    info = L.gemm_plan(a, w, out=out, dropout_p=p)
    assert info.kernel == kernel, f"{name}: expected GEMM kernel {kernel}, the plan says {info.kernel}"
    assert (info.tail_splits > 1) == tail, f"{name}: tail_splits={info.tail_splits}"
    L.gemm(a, w, out=out, dropout_p=p, dropout_seed=SEED, dropout_seed_ptr=sp)
    torch.cuda.synchronize()
    assert_mask((out != 0).cpu().numpy(), keep, f"gemm {name} epilogue mask", ("m", "n"))
    # 2. bias + act + dropout + residual against fp32
    a, w = _operands(dev, M, N, K, lda, g, positive=False)
    bias = torch.randn(N, generator=g).to(dev, torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(dev, torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    info = L.gemm_plan(a, w, out=out, bias=bias, residual=res, act=L.ACT_GELU_TANH, dropout_p=p)
    assert info.kernel == kernel and (info.tail_splits > 1) == tail, (name, info.kernel, info.tail_splits)
    L.gemm(a, w, out=out, bias=bias, act=L.ACT_GELU_TANH, residual=res, dropout_p=p, dropout_seed=SEED, dropout_seed_ptr=sp)
    kt = torch.from_numpy(keep).to(dev)
    ref = res.float() + kt * dscale * F.gelu(a.float() @ w.float().t() + bias.float(), approximate="tanh")
    dropped = ~kt
    assert torch.equal(out[dropped].view(torch.int16), res[dropped].view(torch.int16)), \
        f"gemm {name}: where dropped, out must equal the residual bit for bit"
    err = rel(out, ref)
    print(f"[dropout] gemm {name}: rel-L2 {err:.2e}, worst row {row_err(out, ref):.2e}")
    assert err < 6e-3, f"gemm {name}: rel-L2 {err:.3e}"


# ============================================== attention =============================================================
def _tmap_ok(t, L_):
    """tmap_strides_ok of csrc/attention.cu for a [B, L, H, 64] view."""
    B, _, H, _ = t.shape
    sb, ss, sh = t.stride(0), t.stride(1), t.stride(2)
    if ss <= 0 or sh <= 0 or ss == sh or (B > 1 and sb <= 0):
        return False
    return (sh >= 64 and ss >= sh * H) if sh < ss else (ss >= 64 and sh >= ss * L_)


def attn_paths(q, k, v, d_o):
    """Which kernels dvla_attn_fwd / dvla_attn_bwd pick with dropout on (the short-sequence kernels of
    attention_small.cu take no dropout): 'wgmma' or 'mma.sync' for the forward and for the backward."""
    Lq, Lk = q.shape[1], k.shape[1]
    fwd = Lq >= 96 and _tmap_ok(q, Lq) and _tmap_ok(k, Lk) and _tmap_ok(v, Lk)
    bwd = Lq >= 96 and Lk >= 96 and _tmap_ok(q, Lq) and _tmap_ok(d_o, Lq) and _tmap_ok(k, Lk) and _tmap_ok(v, Lk)
    return ("wgmma" if fwd else "mma.sync"), ("wgmma" if bwd else "mma.sync")


def _random_mask(Lq, Lk, g):
    m = torch.rand(Lq, Lk, generator=g) < 0.3
    m[:, 0] = True
    m[: Lq // 2, 64:128] = False          # skipped tiles
    m[Lq // 2:, 64:128] = True            # full tiles
    return m


def _gpt2_mask(S, num_B, n_obs):
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    add = generate_attention_mask(K=S, num_A=36, num_B=num_B, atten_goal=0, atten_goal_state=False, atten_only_obs=False,
                                  attn_robot_proprio_state=False, mask_l_obs_ratio=0.0, num_obs_token=n_obs,
                                  action_pred_steps=3)
    return add == 0


def _grouped_masks():
    """The grouped token order [A | queries | action] of the GPT-2 step (S = 10): a (1260 x 360) call and a (30 x 1260) one."""
    S, n_a, n_q, n_act = 10, 36, 90, 3
    step_a = torch.arange(S).repeat_interleave(n_a)
    step_q = torch.arange(S).repeat_interleave(n_q)
    rows_step = torch.cat((step_a, step_q))
    main = rows_step[:, None] >= step_a[None, :]
    step_act = torch.arange(S).repeat_interleave(n_act)
    act = torch.cat((step_act[:, None] >= step_a[None, :], step_act[:, None] == step_q[None, :]), dim=1)
    return main, act


# (id, B, H, Lq, Lk, layout, mask, ramp, p, expected (fwd, bwd) kernels)
#   layout: "plain" separate q/k/v; "fused" slices of one [B, L, 3, H, 64] buffer; "bcast" K/V with batch stride 0;
#   "grouped_main" / "grouped_act" the two calls of the grouped GPT-2 form, slices of a fused L = 1290 buffer
ATTN_CASES = [
    ("dit_2x3x6x6", 2, 3, 6, 6, "plain", None, 0.0, 0.1, ("mma.sync", "mma.sync")),
    ("2x2x33x40", 2, 2, 33, 40, "plain", None, 0.0, 0.1, ("mma.sync", "mma.sync")),
    ("3x2x10x265", 3, 2, 10, 265, "plain", None, 0.0, 0.1, ("mma.sync", "mma.sync")),
    ("2x2x64x64", 2, 2, 64, 64, "plain", None, 0.0, 0.5, ("mma.sync", "mma.sync")),
    ("1x2x300x40", 1, 2, 300, 40, "plain", None, 0.0, 0.1, ("wgmma", "mma.sync")),
    ("2x2x130x90", 2, 2, 130, 90, "plain", None, 0.0, 0.1, ("wgmma", "mma.sync")),
    ("1x2x128x128", 1, 2, 128, 128, "plain", None, 0.0, 0.1, ("wgmma", "wgmma")),
    ("1x2x257x517_ramp", 1, 2, 257, 517, "plain", None, 3.0, 0.1, ("wgmma", "wgmma")),
    ("fused_2x2x197", 2, 2, 197, 197, "fused", None, 0.0, 0.1, ("wgmma", "wgmma")),
    ("random_mask_2x2x300x260_ramp", 2, 2, 300, 260, "plain", "random", 3.0, 0.1, ("wgmma", "wgmma")),
    ("random_mask_2x2x80x200", 2, 2, 80, 200, "plain", "random", 0.0, 0.1, ("mma.sync", "mma.sync")),
    ("gpt2_mask_C3_2x2x273", 2, 2, 273, 273, "fused", "c3", 0.0, 0.1, ("wgmma", "wgmma")),
    ("gpt2_mask_C2_1x2x1290", 1, 2, 1290, 1290, "fused", "c2", 0.0, 0.1, ("wgmma", "wgmma")),
    ("grouped_1260x360", 1, 2, 1260, 360, "grouped_main", "grouped_main", 0.0, 0.1, ("wgmma", "wgmma")),
    ("grouped_30x1260", 1, 2, 30, 1260, "grouped_act", "grouped_act", 0.0, 0.1, ("mma.sync", "mma.sync")),
    ("bcast_kv_2x2x130x300", 2, 2, 130, 300, "bcast", None, 0.0, 0.1, ("mma.sync", "mma.sync")),
]


class AttnCase:
    def __init__(self, spec, dev):
        from dreamvla_b200 import ops
        self.name, B, H, Lq, Lk, layout, mask, self.ramp, self.p, self.paths = spec
        self.B, self.H, self.Lq, self.Lk, self.dev = B, H, Lq, Lk, dev
        g = torch.Generator(device="cpu").manual_seed(B * 1000003 + Lq * 1009 + Lk)
        self.g = g
        vis = None
        if mask == "random":
            vis = _random_mask(Lq, Lk, g)
        elif mask == "c3":
            vis = _gpt2_mask(7, 3, 0)
        elif mask == "c2":
            vis = _gpt2_mask(10, 93, 90)
        elif mask in ("grouped_main", "grouped_act"):
            vis = _grouped_masks()[0 if mask == "grouped_main" else 1]
        if vis is not None:
            assert vis.shape == (Lq, Lk) and bool(vis.any(1).all())
        self.vis = vis
        self.mask = ops.AttnMask(vis, dev) if vis is not None else None
        if mask == "random" and Lq >= 256:
            assert {0, 1, 2} <= set(self.mask.flags.flatten().tolist()), "want skipped, partial and full tiles"
        bf = dict(device=dev, dtype=torch.bfloat16)
        if layout in ("fused", "grouped_main", "grouped_act"):
            Lf = 1290 if layout.startswith("grouped") else Lq
            self.buf = torch.zeros(B, Lf, 3, H, 64, **bf)
            qs, ks = {"fused": (slice(None), slice(None)), "grouped_main": (slice(0, 1260), slice(0, 360)),
                      "grouped_act": (slice(1260, 1290), slice(0, 1260))}[layout]
            self.q, self.k, self.v = self.buf[:, qs, 0], self.buf[:, ks, 1], self.buf[:, ks, 2]
        elif layout == "bcast":
            self.q = torch.zeros(B, Lq, H, 64, **bf)
            kv = torch.zeros(2, 1, Lk, H, 64, **bf)
            self.k, self.v = kv[0].expand(B, -1, -1, -1), kv[1].expand(B, -1, -1, -1)
            assert self.k.stride(0) == 0
        else:
            self.q, self.k, self.v = (torch.zeros(B, n, H, 64, **bf) for n in (Lq, Lk, Lk))
        self.d_o = torch.zeros(B, Lq, H, 64, **bf)
        self.dq, self.dk, self.dv = (torch.empty(B, n, H, 64, **bf) for n in (Lq, Lk, Lk))

    @staticmethod
    def _writable(t):
        return t[:1] if t.stride(0) == 0 else t

    def fill_random(self):
        g = self.g
        for t in (self.q, self.k, self.v, self.d_o):
            w = self._writable(t)
            w.copy_(torch.randn(w.shape, generator=g))
        if self.ramp:   # key norms grow along the sequence: the running row maximum keeps rising
            w = self._writable(self.k)
            w.copy_(w.float() * (1.0 + self.ramp * torch.arange(self.Lk, device=self.dev).view(1, -1, 1, 1) / self.Lk))
            self.q.mul_(2.0)

    def bits_flags(self):
        return (self.mask.bits, self.mask.flags) if self.mask is not None else (None, None)

    def visible(self):
        return np.ones((self.Lq, self.Lk), bool) if self.vis is None else self.vis.numpy()

    def fwd(self, L, seed, ctr):
        bits, flags = self.bits_flags()
        return L.attn_fwd(self.q, self.k, self.v, SCALE, bits, flags, dropout_p=self.p, dropout_seed=seed,
                          dropout_seed_ptr=ctr)

    def bwd(self, L, o, lse, seed, ctr):
        bits, flags = self.bits_flags()
        L.attn_bwd(self.q, self.k, self.v, o, self.d_o, lse, SCALE, self.dq, self.dk, self.dv, bits, flags,
                   dropout_p=self.p, dropout_seed=seed, dropout_seed_ptr=ctr)


@pytest.fixture(params=ATTN_CASES, ids=[c[0] for c in ATTN_CASES])
def attn_case(request, dev, L):
    c = AttnCase(request.param, dev)
    assert attn_paths(c.q, c.k, c.v, c.d_o) == c.paths, f"{c.name}: dispatch would run {attn_paths(c.q, c.k, c.v, c.d_o)}"
    return c


def test_attention_dropout_masks_exact(attn_case, L):
    """Forward and dK/dV-backward masks, extracted exactly, equal keep_attn(seed + counter) & visible."""
    c = attn_case
    ctr = WRAP
    sp = counter(ctr, c.dev)
    want = R.keep_attn(SEED, c.B, c.H, c.Lq, c.Lk, c.p, counter=ctr) & c.visible()[None, None]
    c.q.zero_()                                   # P uniform over the visible keys of each row
    vw = c._writable(c.v)
    # forward: V one-hot on a 64-key window -> O[i, c] != 0 <=> key j0 + c kept and visible
    got = np.zeros_like(want)
    for j0 in range(0, c.Lk, 64):
        w = min(64, c.Lk - j0)
        vw.zero_()
        idx = torch.arange(w, device=c.dev)
        vw[:, j0 + idx, :, idx] = 1.0
        o, _ = c.fwd(L, SEED, sp)
        got[:, :, :, j0:j0 + w] = (o.permute(0, 2, 1, 3)[..., :w] != 0).cpu().numpy()
    assert_mask(got, want, f"attention forward ({c.paths[0]}) {c.name}", ("b", "h", "i", "j"))
    # backward dK/dV: dO one-hot on a 64-query window -> dV[j, c] != 0 <=> (i0 + c, j) kept and visible
    vw.zero_()
    o, lse = c.fwd(L, SEED, sp)
    got = np.zeros_like(want)
    for i0 in range(0, c.Lq, 64):
        w = min(64, c.Lq - i0)
        c.d_o.zero_()
        idx = torch.arange(w, device=c.dev)
        c.d_o[:, i0 + idx, :, idx] = 1.0
        c.bwd(L, o, lse, SEED, sp)
        got[:, :, i0:i0 + w, :] = (c.dv.permute(0, 2, 3, 1)[:, :, :w, :] != 0).cpu().numpy()
    assert_mask(got, want, f"attention backward dK/dV ({c.paths[1]}) {c.name}", ("b", "h", "i", "j"))


def _attn_ref(c, keep, dscale):
    """fp32 O = (softmax(S, masked) * keep * scale) @ V, its lse, and dQ, dK, dV by autograd through that expression."""
    q, k, v = (t.detach().float().requires_grad_(True) for t in (c.q, c.k, c.v))
    qh, kh, vh = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * SCALE
    if c.vis is not None:
        s = s.masked_fill(~c.vis.to(c.dev), float("-inf"))
    lse = torch.logsumexp(s, -1)
    pd = s.softmax(-1) * keep * dscale
    o = (pd @ vh).permute(0, 2, 1, 3)
    o.backward(c.d_o.float())
    return o.detach(), lse.detach(), q.grad, k.grad, v.grad


def _attn_bwd_ref(c, o, keep, dscale):
    """The backward as the kernels define it (FlashAttention-2), in fp32: dS = P * (dP * keep * scale - delta) with
    delta = rowsum(dO * O) of the O the backward is GIVEN.  With `o` the kernel's bf16 output this is the same operation
    as the kernels' up to fp32 rounding; autograd's delta uses the unrounded O, which on rows where one key takes nearly
    all of the probability (ramp inputs) leaves dQ and dK a difference of two nearly equal numbers, dominated by O's bf16
    rounding -- fine for a whole-tensor bar, not for a per-row one."""
    qh, kh, vh, doh, oh = (t.float().permute(0, 2, 1, 3) for t in (c.q, c.k, c.v, c.d_o, o))
    s = (qh @ kh.transpose(-1, -2)) * SCALE
    if c.vis is not None:
        s = s.masked_fill(~c.vis.to(c.dev), float("-inf"))
    p = s.softmax(-1)
    dv = (p * keep * dscale).transpose(-1, -2) @ doh
    ds = p * ((doh @ vh.transpose(-1, -2)) * keep * dscale - (doh * oh).sum(-1, keepdim=True))
    dq, dk = (ds @ kh) * SCALE, (ds.transpose(-1, -2) @ qh) * SCALE
    return tuple(t.permute(0, 2, 1, 3) for t in (dq, dk, dv))


def test_attention_dropout_numerics(attn_case, L):
    """O, lse, dQ, dK, dV against fp32 softmax(S) * keep * scale @ V and its autograd (whole tensor), and per row against
    the same expression with the backward's delta taken from the kernel's O; the per-row dQ bar is what pins the dQ
    kernel's own regeneration of the mask."""
    c = attn_case
    ctr = 987654321
    sp = counter(ctr, c.dev)
    c.fill_random()
    keep = torch.from_numpy(R.keep_attn(SEED, c.B, c.H, c.Lq, c.Lk, c.p, counter=ctr)).to(c.dev)
    _, dscale = R.thresh_scale(c.p)
    o, lse = c.fwd(L, SEED, sp)
    # the counter is only added to the seed: the same call with the sum as the seed and no counter is bit-identical
    o2, _ = c.fwd(L, (SEED + ctr) % 2 ** 64, None)
    assert torch.equal(o, o2), "dropout_seed_ptr = c must draw the mask of dropout_seed + c"
    c.bwd(L, o, lse, SEED, sp)
    torch.cuda.synchronize()
    o_ref, lse_ref, dq_ref, dk_ref, dv_ref = _attn_ref(c, keep, dscale)
    # the explicit backward with the fp32 O is autograd's, which checks the formula the per-row references use
    for mine, ag in zip(_attn_bwd_ref(c, o_ref, keep, dscale), (dq_ref, dk_ref, dv_ref)):
        assert rel(mine, ag) < 1e-4
    rows = dict(zip(("dq", "dk", "dv"), _attn_bwd_ref(c, o, keep, dscale)))
    lse_err = float((lse - lse_ref).abs().max())
    errs = {"o": (rel(o, o_ref), row_err(o, o_ref))}
    for name, got, ref in (("dq", c.dq, dq_ref), ("dk", c.dk, dk_ref), ("dv", c.dv, dv_ref)):
        errs[name] = (rel(got, ref), row_err(got, rows[name]))
    print(f"[dropout] attn {c.name} fwd={c.paths[0]} bwd={c.paths[1]} lse {lse_err:.1e} " +
          " ".join(f"{k} {e:.1e}/row {r:.1e}" for k, (e, r) in errs.items()))
    assert lse_err < 1e-3, f"lse must be the logsumexp of the masked scores (dropout does not change it): {lse_err:.3e}"
    bars = {"o": (6e-3, 2e-2), "dq": (1e-2, 3e-2), "dk": (1e-2, 3e-2), "dv": (1e-2, 3e-2)}
    bad = {k: e for k, e in errs.items() if not (e[0] < bars[k][0] and e[1] < bars[k][1])}
    assert not bad, f"{c.name}: (rel-L2, worst row) over the bars {bars}: {bad}"


# ============================================== seeds, CUDA graphs, errors ============================================
def test_cuda_graph_replays_draw_the_counters_masks(dev, L):
    """One graph with dvla_dropout, an attention forward and a dropout GEMM, all reading the seed counter; every replay
    draws the masks of the counter value it runs with (seeds baked into the graph, the counter advanced on the device)."""
    g = torch.Generator(device="cpu").manual_seed(17)
    p, sd, sa, sg = 0.1, SEED, SEED ^ 0xFFFF, SEED + 1
    ctr = counter(2 ** 64 - 2, dev)
    x = (torch.randn(24, 1000, generator=g) + 0.01).to(dev, torch.bfloat16)
    y = torch.empty_like(x)
    a = (torch.rand(256, 128, generator=g) + 0.1).to(dev, torch.bfloat16)
    w = (torch.rand(136, 128, generator=g) + 0.1).to(dev, torch.bfloat16)
    gout = torch.empty(256, 136, device=dev, dtype=torch.bfloat16)
    B, H, Lq, Lk = 1, 2, 128, 64
    q = torch.zeros(B, Lq, H, 64, device=dev, dtype=torch.bfloat16)
    k = torch.randn(B, Lk, H, 64, generator=g).to(dev, torch.bfloat16)
    v = torch.zeros(B, Lk, H, 64, device=dev, dtype=torch.bfloat16)
    idx = torch.arange(64, device=dev)
    v[:, idx, :, idx] = 1.0

    def run():
        L.dropout(x, p, sd, out=y, seed_ptr=ctr)
        L.gemm(a, w, out=gout, dropout_p=p, dropout_seed=sg, dropout_seed_ptr=ctr)
        return L.attn_fwd(q, k, v, SCALE, dropout_p=p, dropout_seed=sa, dropout_seed_ptr=ctr)[0]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()                                     # workspace, kernel attributes: set up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        o = run()
    for r in range(3):
        c = (2 ** 64 - 2 + r) % 2 ** 64           # 2^64 - 2, 2^64 - 1, 0
        graph.replay()
        torch.cuda.synchronize()
        assert_mask((y != 0).cpu().numpy(), R.keep_rows(sd, 24, 1000, p, counter=c), f"graph replay {r} dvla_dropout",
                    ("row", "col"))
        assert_mask((gout != 0).cpu().numpy(), R.keep_rows(sg, 256, 136, p, counter=c), f"graph replay {r} GEMM",
                    ("m", "n"))
        assert_mask((o.permute(0, 2, 1, 3) != 0).cpu().numpy(), R.keep_attn(sa, B, H, Lq, Lk, p, counter=c),
                    f"graph replay {r} attention", ("b", "h", "i", "j"))
        ctr.add_(1)


@pytest.mark.parametrize("p", [float("nan"), 1.0, 1.5, -0.25])
def test_dropout_p_out_of_range_is_rejected_before_any_launch(dev, L, p):
    x = torch.randn(64, 64, device=dev).to(torch.bfloat16)
    q = torch.randn(1, 128, 2, 64, device=dev).to(torch.bfloat16)
    o, lse = L.attn_fwd(q, q, q, SCALE)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    L.gemm_workspace(dev)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    calls = {
        "attn_fwd": lambda: L.attn_fwd(q, q, q, SCALE, dropout_p=p, dropout_seed=1),
        "attn_bwd": lambda: L.attn_bwd(q, q, q, o, q, lse, SCALE, dq, dk, dv, dropout_p=p, dropout_seed=1),
        "gemm": lambda: L.gemm(x, x, dropout_p=p, dropout_seed=1),
        "dropout": lambda: L.dropout(x, p, 1),
    }
    for name, fn in calls.items():
        with pytest.raises(RuntimeError, match="out of range"):
            fn()
        assert L.launch_count() == n0, f"{name} launched a kernel with dropout_p={p}"


# ============================================== GPT-2 backbone in train mode ==========================================
def _gpt2_ref(P, x, vis, keeps, dscale, n_layer, H):
    """fp32 GPT-2 backbone (gpt2.py): embedding dropout, then per block h += drop(c_proj(attn(LN1 h))) with dropout on the
    attention probabilities, h += drop(MLP(LN2 h)); LN_f."""
    B, Lx, D = x.shape
    ln = lambda t, n: F.layer_norm(t, (D,), P[n + ".weight"], P[n + ".bias"], 1e-5)     # noqa: E731
    h = x * keeps[0] * dscale
    for i in range(n_layer):
        pre, (ka, kp, km) = f"h.{i}.", keeps[1 + 3 * i: 4 + 3 * i]
        qkv = (ln(h, pre + "ln_1") @ P[pre + "attn.c_attn.weight"] + P[pre + "attn.c_attn.bias"]).view(B, Lx, 3, H, 64)
        q, k, v = (qkv[:, :, t].transpose(1, 2) for t in range(3))
        s = ((q @ k.transpose(-1, -2)) * SCALE).masked_fill(~vis, float("-inf"))
        o = ((s.softmax(-1) * ka * dscale) @ v).transpose(1, 2).reshape(B, Lx, D)
        h = h + (o @ P[pre + "attn.c_proj.weight"] + P[pre + "attn.c_proj.bias"]) * kp * dscale
        f = F.gelu(ln(h, pre + "ln_2") @ P[pre + "mlp.c_fc.weight"] + P[pre + "mlp.c_fc.bias"], approximate="tanh")
        h = h + (f @ P[pre + "mlp.c_proj.weight"] + P[pre + "mlp.c_proj.bias"]) * km * dscale
    return ln(h, "ln_f")


def test_gpt2_backbone_train_mode_with_dropout(dev, L, monkeypatch):
    from dreamvla_b200 import ops
    from dreamvla_b200.models.gpt2 import GPT2Config, GPT2Model
    n_layer, D, H, B = 2, 1024, 16, 2
    p = 0.1
    torch.manual_seed(0)
    model = GPT2Model(GPT2Config(hidden_size=D, n_layer=n_layer, n_head=H, resid_pdrop=p, embd_pdrop=p, attn_pdrop=p))
    with torch.no_grad():
        for name, prm in model.named_parameters():
            if name.endswith("bias"):
                prm.normal_(0.0, 0.05)
            elif "ln" in name:
                prm.normal_(1.0, 0.1)
    model = model.bfloat16().to(dev).train()
    vis = _gpt2_mask(7, 3, 0)
    Lx = vis.shape[0]
    mask = ops.AttnMask(vis, dev)
    g = torch.Generator(device="cpu").manual_seed(3)
    x = torch.randn(B, Lx, D, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    gy = torch.randn(B, Lx, D, generator=g).to(dev)

    seeds = []
    real_next_seed = ops.next_seed

    def recording_next_seed():
        seeds.append(real_next_seed())
        return seeds[-1]

    monkeypatch.setattr(ops, "next_seed", recording_next_seed)
    ctr_t = ops.seed_counter(dev)
    saved = ctr_t.clone()
    ctr = 2 ** 64 - 1000                      # the effective seeds wrap past 2^64
    ctr_t.copy_(counter(ctr, dev))
    try:
        out = model(attention_mask=mask, inputs_embeds=x)
        (out.float() * gy).sum().backward()
        torch.cuda.synchronize()
    finally:
        ctr_t.copy_(saved)
    assert len(seeds) == 1 + 3 * n_layer, f"expected one seed for the embedding and three per block, got {len(seeds)}"

    # restated masks: embedding, then per block attention probabilities, c_proj residual, MLP residual
    rows = B * Lx
    keeps = [torch.from_numpy(R.keep_rows(seeds[0], rows, D, p, counter=ctr)).view(B, Lx, D)]
    for i in range(n_layer):
        sa, sp_, sm = seeds[1 + 3 * i: 4 + 3 * i]
        keeps += [torch.from_numpy(R.keep_attn(sa, B, H, Lx, Lx, p, counter=ctr)),
                  torch.from_numpy(R.keep_rows(sp_, rows, D, p, counter=ctr)).view(B, Lx, D),
                  torch.from_numpy(R.keep_rows(sm, rows, D, p, counter=ctr)).view(B, Lx, D)]
    keeps = [k.to(dev) for k in keeps]
    _, dscale = R.thresh_scale(p)
    P = {n: prm.detach().float().requires_grad_(True) for n, prm in model.named_parameters()}
    xr = x.detach().float().requires_grad_(True)
    ref = _gpt2_ref(P, xr, vis.to(dev), keeps, dscale, n_layer, H)
    (ref * gy).sum().backward()

    errs = [("output", rel(out, ref)), ("d inputs_embeds", rel(x.grad, xr.grad))]
    errs += [(n, rel(prm.grad, P[n].grad)) for n, prm in model.named_parameters()]
    for n, e in errs:
        print(f"[dropout] gpt2 {n}: rel-L2 {e:.2e}")
    assert errs[0][1] < 2e-2, f"output rel-L2 {errs[0][1]:.3e}"
    bad = [(n, e) for n, e in errs[1:] if not e < 6e-2]
    assert not bad, f"gradient mismatch under the restated dropout masks: {bad}"
