"""Every dvla_gemm path and epilogue checked element by element against an fp64 reference, with guard bands.

Each case of tests/gemm_cases.py (path x majorness x epilogue recipe x edge shape, distinct row strides) is run once:
  * path: the live plan (real pointers, this device) is the path the case declares;
  * guard bands: out, aux_out and the residual are windows of larger buffers filled with a signalling-NaN pattern no kernel
    writes (bf16 0x7FA1, fp32 0x7FA1A1A1).  Every element outside the [M, N] window must be bit-unchanged afterwards, every
    input (a, b, bias, aux_in, a separate residual) too, and the workspace's arrival counters must be zero again;
  * values: every element of out (and of aux_out) within the bound below;
  * bits: a second launch on the restored buffers gives the same bits on every path but split-K (bf16 atomics land in
    any order) -- the K-split tail included, since its splits are summed in a fixed order.
and three properties: rows of a sub-wave GEMM do not depend on the other rows of the call, a whole-tile plan gives the same
bits under any SM budget, and the split-K weight gradients stay within their bound.

The bound.  With S = |alpha| sum_k |a_k b_k| + |bias| (in fp64), the fp32 value the epilogue starts from differs from
alpha.A.B^T + bias by at most (K + 2) 2^-23 S: the products of bf16 operands are exact in fp32, each of the K - 1
additions of the accumulation (tensor-core or FMA, in any order, with round-to-nearest or truncation) costs at most
2^-23 of the running |sum| <= S, and the alpha scaling and the bias add one rounding each.  The epilogue then
  * applies act or multiplies by act'(aux_in): an error d of its input becomes at most c_act d with c_act = 1.2 >= max|act'|
    (GELU 1.13, SiLU 1.10, QuickGELU 1.10, ReLU / none 1) -- the dgrad multiplies by act'(x) with |act'(x)| <= c_act;
  * evaluates act / act' with ex2.approx, rcp.approx (relative errors ~2^-22, 2^-23) and the Abramowitz-Stegun erf
    (1.5e-7 absolute) in a few fp32 operations (csrc/common.cuh): at most e_act |pre| for act(pre), and e_act (1 + |x|) |v|
    for v act'(x), with e_act = 2^-18 (about 8x the sum of those errors).  ReLU and none are exact up to fp32 rounding,
    e_act = 2^-22 there, which also covers the roundings of the dropout scale and of the residual add;
  * scales kept elements by the dropout scale s = 1/(1 - p) (both error terms grow by s);
  * rounds once to the output type: u_out |ref| (u_out = 2^-8 bf16, 2^-24 fp32), applied to a value within the terms above.
So every element must satisfy
    |got - ref| <= u_out |ref| + (1 + u_out) s (c_act (K + 2) 2^-23 S + e_act-term).
aux_out (the pre-activation, bf16) is checked against alpha.A.B^T + bias with u_out = 2^-8 and no activation terms.
Split-K adds each split's partial with one bf16 red.global.add: the partials are rounded to bf16 (<= 2^-8 S together) and
each of the k_splits adds rounds the running value (<= 2^-8 (|G0| + S)), so (k_splits + 1) 2^-8 (|G0| + S) more.
The worst err / bound of each case is printed.
"""
import math
import zlib

import pytest
import torch

from tests import gemm_cases as GC
from tests import philox_ref as R

pytestmark = pytest.mark.gpu

SEED = 0xC0FFEE1234567890
CTR = 2 ** 64 - 5                    # SEED + CTR wraps past 2^64
SENT = {False: (0x7FA1, torch.int16, torch.bfloat16), True: (0x7FA1A1A1, torch.int32, torch.float32)}
C_ACT = 1.2
APPROX_ACTS = (1, 2, 3, 5)


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
    v = int(value) % 2 ** 64
    return torch.tensor([v - 2 ** 64 if v >= 2 ** 63 else v], dtype=torch.int64, device=dev)


def sentinel(n, fp32, dev):
    pat, ity, fty = SENT[fp32]
    return torch.full((n,), pat, dtype=ity, device=dev).view(fty)


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def window(buf, rows, cols, ld, off):
    return buf.as_strided((rows, cols), (ld, 1), off)


def span(rows, ld, off):
    """Buffer length for a [rows, ld] window at element offset off, plus two guard rows."""
    return off + (rows + 2) * ld


def randn(g, n, scale, dev, dtype=torch.bfloat16):
    return (torch.randn(n, generator=g, device=dev) * scale).to(dtype)


def act_fwd(x, act):
    if act == 1:
        return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2)))
    if act == 2:
        return 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3)))
    if act == 3:
        return x * torch.sigmoid(1.702 * x)
    if act == 4:
        return torch.clamp_min(x, 0)
    if act == 5:
        return x * torch.sigmoid(x)
    return x


def act_grad(x, act):
    if act == 1:
        return 0.5 * (1 + torch.special.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    if act == 2:
        k = math.sqrt(2 / math.pi)
        t = torch.tanh(k * (x + 0.044715 * x ** 3))
        return 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * k * (1 + 3 * 0.044715 * x * x)
    if act == 3:
        s = torch.sigmoid(1.702 * x)
        return s + 1.702 * x * s * (1 - s)
    if act == 4:
        return (x > 0).double()
    if act == 5:
        s = torch.sigmoid(x)
        return s + x * s * (1 - s)
    return torch.ones_like(x)


def check_bound(what, got, ref, bound):
    """Every element within its bound (a NaN fails); returns the worst err / bound."""
    diff = (got.double() - ref).abs()
    ok = diff <= bound
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:6].tolist()
        ex = "; ".join(f"[{r},{c}] got={float(got[r, c]):.6g} ref={float(ref[r, c]):.6g} bound={float(bound[r, c]):.3g}"
                       for r, c in bad)
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements outside the bound, e.g. {ex}")
    return float((diff / bound.clamp_min(1e-300)).max())


def assert_guard(what, buf, before, win_mask):
    """Everything of `buf` outside the window bit-identical to `before`."""
    changed = (bits(buf) != bits(before)) & ~win_mask
    if bool(changed.any()):
        idx = changed.nonzero()[:6].flatten().tolist()
        raise AssertionError(f"{what}: {int(changed.sum())} elements outside the [M, N] window were written, e.g. at {idx}")


def win_mask(n, rows, cols, ld, off, dev):
    m = torch.zeros(n, dtype=torch.bool, device=dev)
    window(m, rows, cols, ld, off).fill_(True)
    return m


class Run:
    """Buffers, call and fp64 reference of one case."""

    def __init__(self, c, dev, seed):
        self.c, self.dev = c, dev
        g = torch.Generator(device=dev).manual_seed(seed)
        M, N, K = c.M, c.N, c.K
        ar, ac = (K, M) if c.a_mn else (M, K)
        br, bc = (K, N) if c.b_mn else (N, K)
        self.abuf = randn(g, span(ar, c.lda, c.a_off), 0.5, dev)
        self.bbuf = randn(g, span(br, c.ldb, c.b_off), 1.0 / math.sqrt(K), dev)
        self.a = window(self.abuf, ar, ac, c.lda, c.a_off)
        self.b = window(self.bbuf, br, bc, c.ldb, c.b_off)
        self.A = self.a.t() if c.a_mn else self.a          # logical [M, K] / [N, K]
        self.B = self.b.t() if c.b_mn else self.b
        fp32 = c.out_fp32
        odt = torch.float32 if fp32 else torch.bfloat16
        self.obuf = sentinel(span(M, c.ldo, c.out_off), fp32, dev)
        self.out = window(self.obuf, M, N, c.ldo, c.out_off)
        self.bias = randn(g, N, 0.5, dev) if c.has_bias else None
        self.res = self.rbuf = None
        if c.residual_is_out:
            self.out.copy_(randn(g, M * N, 1.0, dev, odt).view(M, N))
            self.res = self.out
        elif c.has_residual:
            self.rbuf = sentinel(span(M, c.ldr, c.res_off), fp32, dev)
            self.res = window(self.rbuf, M, N, c.ldr, c.res_off)
            self.res.copy_(randn(g, M * N, 1.0, dev, odt).view(M, N))
        self.xbuf = self.aux_out = self.aux_in = None
        if c.recipe == "full":
            self.xbuf = sentinel(span(M, c.ld_aux, c.aux_off), False, dev)
            self.aux_out = window(self.xbuf, M, N, c.ld_aux, c.aux_off)
        elif c.recipe == "dgrad":
            self.xbuf = sentinel(span(M, c.ld_aux, c.aux_off), False, dev)
            self.aux_in = window(self.xbuf, M, N, c.ld_aux, c.aux_off)
            self.aux_in.copy_(randn(g, M * N, 1.5, dev).view(M, N))
        self.ctr = counter(CTR, dev) if c.recipe == "dropout" else None
        self.before = {k: v.clone() for k, v in self.buffers().items()}

    def buffers(self):
        d = {"a": self.abuf, "b": self.bbuf, "out": self.obuf}
        for k, v in (("bias", self.bias), ("residual", self.rbuf), ("aux", self.xbuf)):
            if v is not None:
                d[k] = v
        return d

    def kwargs(self):
        c = self.c
        return dict(a_mn=c.a_mn, b_mn=c.b_mn, bias=self.bias, act=c.act, residual=self.res, aux_out=self.aux_out,
                    aux_in=self.aux_in, out=self.out, alpha=c.alpha, dropout_p=GC.DROPOUT_P if self.ctr is not None else 0.0,
                    dropout_seed=SEED, dropout_seed_ptr=self.ctr)

    def restore(self):
        for k, v in self.buffers().items():
            v.copy_(self.before[k])

    def reference(self, k_splits=1):
        """(ref, bound) of out and, with aux_out, (pre, bound) of aux_out: fp64 on the device."""
        c = self.c
        A, B = self.A.double(), self.B.double()
        acc = A @ B.t()
        S = abs(c.alpha) * (A.abs() @ B.abs().t())
        pre = c.alpha * acc
        if self.bias is not None:
            b = self.bias.double()
            pre, S = pre + b, S + b.abs()
        acc_term = (c.K + 2) * 2.0 ** -23 * S
        e_act = 2.0 ** -18 if c.act in APPROX_ACTS else 2.0 ** -22
        if self.aux_in is not None:
            x = self.aux_in.double()
            y = pre * act_grad(x, c.act)
            eps = e_act * (1 + x.abs()) * pre.abs()
        else:
            y = act_fwd(pre, c.act)
            eps = e_act * pre.abs()
        scale = 1.0
        if self.ctr is not None:
            keep = torch.from_numpy(R.keep_rows(SEED, c.M, c.N, GC.DROPOUT_P, counter=CTR)).to(self.dev)
            _, scale = R.thresh_scale(GC.DROPOUT_P)
            y = torch.where(keep, y * scale, torch.zeros_like(y))
        g0 = None
        if self.res is not None:
            g0 = self.before["out" if c.residual_is_out else "residual"]
            g0 = window(g0, c.M, c.N, c.ldo if c.residual_is_out else c.ldr,
                        c.out_off if c.residual_is_out else c.res_off).double()
            y = y + g0
        u = 2.0 ** -24 if c.out_fp32 else 2.0 ** -8
        bound = u * y.abs() + (1 + u) * scale * (C_ACT * acc_term + eps)
        if k_splits > 1:
            bound = bound + (k_splits + 1) * 2.0 ** -8 * (g0.abs() + S)
        aux = None
        if self.aux_out is not None:
            aux = (pre, 2.0 ** -8 * pre.abs() + (1 + 2.0 ** -8) * acc_term)
        return y, bound, aux


def run_case(L, dev, c, seed):
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    r = Run(c, dev, seed)
    info = L.gemm_plan(r.a, r.b, **r.kwargs())
    got_path = GC.path_of(info, c)
    assert got_path == c.path_at(sms), f"{c.id}: plans {got_path} on {sms} SMs, the table says {c.path_at(sms)}"
    L.gemm(r.a, r.b, **r.kwargs())
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in r.buffers().items()}
    # guard bands and inputs
    for k in ("a", "b", "bias", "residual") + (("aux",) if r.aux_in is not None else ()):
        if k in first:
            assert torch.equal(bits(first[k]), bits(r.before[k])), f"{c.id}: input {k} was modified"
    n = r.obuf.numel()
    assert_guard(f"{c.id}: out", r.obuf, r.before["out"], win_mask(n, c.M, c.N, c.ldo, c.out_off, dev))
    if r.aux_out is not None:
        assert_guard(f"{c.id}: aux_out", r.xbuf, r.before["aux"],
                     win_mask(r.xbuf.numel(), c.M, c.N, c.ld_aux, c.aux_off, dev))
    ws = L.gemm_workspace(dev)
    assert int(ws[:65536].count_nonzero()) == 0, f"{c.id}: workspace arrival counters left non-zero"
    # values
    ref, bound, aux = r.reference(info.k_splits if info.atomic_out else 1)
    worst = check_bound(f"{c.id}: out", r.out, ref, bound)
    msg = f"[gemm-paths] {c.id}: worst err/bound out {worst:.3f}"
    if aux is not None:
        msg += f", aux_out {check_bound(f'{c.id}: aux_out', r.aux_out, *aux):.3f}"
    print(msg)
    return r, info, first


@pytest.mark.parametrize("case", GC.CASES, ids=[c.id for c in GC.CASES])
def test_gemm_path(dev, L, case):
    r, info, first = run_case(L, dev, case, seed=zlib.crc32(case.id.encode()))
    if info.atomic_out:
        return
    r.restore()
    L.gemm(r.a, r.b, **r.kwargs())
    torch.cuda.synchronize()
    for k, v in r.buffers().items():
        assert torch.equal(bits(v), bits(first[k])), f"{case.id}: a second launch changed the bits of {k}"


# ============================================== properties ============================================================
def _sub_wave(info):
    return info.kernel == 2 and info.tail_splits <= 1 and info.k_splits == 1


@pytest.mark.parametrize("M,N,K,b_mn", [(300, 768, 3072, False), (260, 1024, 1024, True)])
def test_row_batch_invariance(dev, L, M, N, K, b_mn):
    """Rows [r0, r0 + m) of an M-row sub-wave GEMM equal the m-row GEMM of the same A rows bit for bit (the incremental
    rollout recomputes only new rows and relies on this)."""
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    a = randn(g, M * K, 0.5, dev).view(M, K)
    w = randn(g, N * K, 1.0 / math.sqrt(K), dev).view(K, N) if b_mn else randn(g, N * K, 1.0 / math.sqrt(K), dev).view(N, K)
    bias = randn(g, N, 0.5, dev)
    res = randn(g, M * N, 1.0, dev).view(M, N)
    kw = dict(b_mn=b_mn, bias=bias, act=2)
    assert _sub_wave(L.gemm_plan(a, w, residual=res, **kw))
    full = L.gemm(a, w, residual=res, **kw)
    for m, r0 in ((1, 131), (7, 5), (129, 64)):
        assert _sub_wave(L.gemm_plan(a[r0:r0 + m], w, residual=res[r0:r0 + m], **kw))
        part = L.gemm(a[r0:r0 + m], w, residual=res[r0:r0 + m], **kw)
        torch.cuda.synchronize()
        assert torch.equal(bits(part), bits(full[r0:r0 + m])), f"rows [{r0}, {r0 + m}) differ from the {M}-row GEMM"


@pytest.mark.parametrize("M,N,K,accum", [(2000, 1024, 320, False), (1104, 776, 512, True)])
def test_sm_budget_same_bits(dev, L, M, N, K, accum):
    """A whole-tile plan computes every tile the same way whatever the grid: the same bits at 40 SMs as on the full GPU."""
    g = torch.Generator(device=dev).manual_seed(M * N)
    a = randn(g, K * M, 0.5, dev).view(K, M) if accum else randn(g, M * K, 0.5, dev).view(M, K)
    w = randn(g, K * N, 1.0 / math.sqrt(K), dev).view(K, N) if accum else randn(g, N * K, 1.0 / math.sqrt(K), dev).view(N, K)
    g0 = randn(g, M * N, 1.0, dev).view(M, N)
    kw = dict(a_mn=True, b_mn=True) if accum else dict(bias=randn(g, N, 0.5, dev), act=1, residual=g0)

    def call():
        out = g0.clone() if accum else torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        extra = dict(residual=out) if accum else {}
        info = L.gemm_plan(a, w, out=out, **kw, **extra)
        assert info.kernel == 2 and info.tail_splits <= 1 and info.k_splits == 1, "not a whole-tile plan"
        L.gemm(a, w, out=out, **kw, **extra)
        torch.cuda.synchronize()
        return info, out

    info_full, full = call()
    prev = L.set_sm_budget(40)
    try:
        info_40, small = call()
    finally:
        L.set_sm_budget(prev)
    assert info_40.grid_ctas <= 40 < info_full.grid_ctas
    assert torch.equal(bits(small), bits(full)), "the SM budget changed the result of a whole-tile GEMM"


@pytest.mark.parametrize("M,N,K", [(3072, 768, 31520), (1024, 1024, 20640), (768, 3072, 3940)])
def test_splitk_weight_gradients(dev, L, M, N, K):
    """Weight-gradient shapes accumulate with uniform split-K and bf16 atomics, within the split-K bound."""
    c = GC.make("wgmma_splitk", M, N, K, True, True, "accum")
    r, info, _ = run_case(L, dev, c, seed=M + N + K)
    assert info.k_splits > 1 and info.atomic_out == 1, (info.k_splits, info.atomic_out)
