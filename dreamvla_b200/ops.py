"""torch.autograd.Function ops backed by libdvla_sm90.so -- the host-side mirror of the reference's PyTorch call sites.

Every op here runs ONLY on the hand-written CUDA kernels (via dreamvla_b200._lib); there is no eager fallback.

Gradient plumbing ("fused wgrad accumulation"): if a parameter carries `_dvla_grad` (a bf16 view into the flat
gradient buffer owned by dreamvla_b200.utils.train_utils.FlatParams) the weight gradient GEMM accumulates straight
into it in its epilogue and autograd receives None; 1-D parameters (biases, LayerNorm affine) accumulate in fp32 into
`_dvla_grad32`.  Without those attributes the ops return ordinary gradient tensors (unit tests, stock optimisers).
"""
from __future__ import annotations

import torch

from . import _lib as L

ACT_IDS = L.ACT_IDS

# ----------------------------------------------------------------------------------------------------------------------
# dropout seeds: one 64-bit counter per process, advanced per op call (fwd stores the seed for the bwd)
# ----------------------------------------------------------------------------------------------------------------------
_seed_state = {"base": 0x243F6A8885A308D3, "ctr": 0}


def manual_seed(seed: int) -> None:
    _seed_state["base"] = (int(seed) * 0x9E3779B97F4A7C15 + 0x632BE59BD9B4E019) & 0xFFFFFFFFFFFFFFFF
    _seed_state["ctr"] = 0


def next_seed() -> int:
    _seed_state["ctr"] += 1
    return (_seed_state["base"] + _seed_state["ctr"] * 0xD1342543DE82EF95) & 0xFFFFFFFFFFFFFFFF


_seed_counters = {}


def seed_counter(device) -> torch.Tensor:
    """Device-resident uint64 counter added to every dropout seed at kernel run time.  The train step increments it on
    the device each step, so CUDA-graph replays (whose host-side seeds are baked in) still draw fresh masks."""
    key = str(device)
    t = _seed_counters.get(key)
    if t is None:
        t = torch.zeros(1, device=device, dtype=torch.int64)
        _seed_counters[key] = t
    return t


def _as2d(x):
    return x.reshape(-1, x.shape[-1])


def _bf16c(x):
    x = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
    return x if x.is_contiguous() else x.contiguous()


def _accum_grad_2d(param, a, b, a_mn, b_mn):
    """dW = A @ B^T into param._dvla_grad (accumulate) or a fresh tensor."""
    gbuf = getattr(param, "_dvla_grad", None)
    if gbuf is not None:
        g2 = gbuf.view(param.shape)
        L.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=g2, residual=g2)
        return None
    return L.gemm(a, b, a_mn=a_mn, b_mn=b_mn)


def _act_bwd_with_bias_grad(dz, aux, act, bias):
    """dz * act'(aux) -> (d_pre, db, done): when the bias owns a flat fp32 gradient slot its gradient (the column sum of
    d_pre) is accumulated by the same kernel (done=True, db=None); otherwise the caller takes the separate column sum."""
    g32 = getattr(bias, "_dvla_grad32", None) if (bias is not None and bias.requires_grad) else None
    if g32 is not None and dz.dim() == 2 and dz.is_contiguous():
        return L.act_bwd(dz, aux, act, colsum_out=g32), True
    return L.act_bwd(dz, aux, act), False


def _accum_bias_grad(param, dy2d):
    g32 = getattr(param, "_dvla_grad32", None)
    if g32 is not None:
        L.colsum_accum(dy2d, g32)
        return None
    tmp = torch.zeros(dy2d.shape[1], device=dy2d.device, dtype=torch.float32)
    L.colsum_accum(dy2d, tmp)
    return tmp.to(torch.bfloat16)


# Function.forward always runs with grad mode off, and ctx.needs_input_grad reports requires_grad of the inputs even under
# torch.no_grad() (frozen ViT / CLIP towers, inference).  The wrappers record the caller's grad mode here so that forward
# only writes and saves backward state (pre-activations, LN stats, LSE) when a backward can actually happen.
_grad_on = True


def _apply(fn, *args):
    global _grad_on
    prev = _grad_on
    _grad_on = torch.is_grad_enabled()
    try:
        return fn.apply(*args)
    finally:
        _grad_on = prev


def on_grad_ready(t: torch.Tensor, callback):
    """Run `callback()` during backward at the moment the gradient w.r.t. `t` is complete, i.e. when every op that consumed
    `t` (and everything downstream of it) has enqueued its backward kernels -- including the fused weight-gradient GEMMs.
    The gradient itself is left untouched."""
    def _hook(grad):
        callback()
        return None
    t.register_hook(_hook)
    return t


class _Linear(torch.autograd.Function):
    """y = dropout(act(x @ W^T + b)) + residual.   weight_kn=False: W is [out,in] (nn.Linear); True: [in,out] (HF Conv1D)."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, act, weight_kn, dropout_p, alpha):
        x2 = _as2d(_bf16c(x))
        N = weight.shape[1] if weight_kn else weight.shape[0]
        need_grad = _grad_on and any(ctx.needs_input_grad)
        aux = None
        if act != 0 and need_grad:
            aux = torch.empty((x2.shape[0], N), device=x2.device, dtype=torch.bfloat16)
        seed = next_seed() if dropout_p > 0 else 0
        res2 = _as2d(_bf16c(residual)) if residual is not None else None
        y = L.gemm(x2, weight, b_mn=weight_kn, bias=bias, act=act, residual=res2, aux_out=aux, alpha=alpha,
                   dropout_p=dropout_p, dropout_seed=seed,
                   dropout_seed_ptr=seed_counter(x2.device) if dropout_p > 0 else None)
        ctx.save_for_backward(x2, aux)
        ctx.weight, ctx.bias = weight, bias
        ctx.meta = (act, weight_kn, dropout_p, seed, alpha, x.shape, residual is not None,
                    residual.shape if residual is not None else None)
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        x2, aux = ctx.saved_tensors
        weight, bias = ctx.weight, ctx.bias
        act, weight_kn, dropout_p, seed, alpha, xshape, has_res, res_shape = ctx.meta
        dy2 = _as2d(_bf16c(dy))
        d_res = dy.view(res_shape) if has_res and ctx.needs_input_grad[3] else None
        dz = dy2  # gradient w.r.t. (act output before dropout)
        if dropout_p > 0:
            dz = L.dropout(dy2, dropout_p, seed, seed_ptr=seed_counter(dy2.device))
        bias_done = False
        if act != 0:                          # gradient w.r.t. the pre-activation (alpha*acc + bias), + the bias gradient
            dz, bias_done = _act_bwd_with_bias_grad(dz, aux, act, bias)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            # dX[M,K] = dZ[M,N] @ W ; contraction over N.  W [N,K] -> B(n_out=k, k_contr=n) = W[n, k]: MN-major B.
            dx = L.gemm(dz, weight, b_mn=not weight_kn, alpha=alpha).view(xshape)
        if weight.requires_grad:
            if weight_kn:   # dW[K,N] = X^T dZ : A = X as [K x M] (mn-major), B = dZ as [N x M] (mn-major)
                dw = _accum_grad_2d(weight, x2, dz, True, True) if alpha == 1.0 else None
            else:           # dW[N,K] = dZ^T X
                dw = _accum_grad_2d(weight, dz, x2, True, True) if alpha == 1.0 else None
            if alpha != 1.0:
                raise RuntimeError("alpha != 1 with trainable weight is not supported")
        if bias is not None and bias.requires_grad and not bias_done:
            db = _accum_bias_grad(bias, dz)
        return dx, dw, db, d_res, None, None, None, None


def linear(x, weight, bias=None, *, act=None, residual=None, weight_kn=False, dropout_p=0.0, alpha=1.0):
    """Fused linear layer on the wgmma GEMM.  x [..., K] bf16."""
    return _apply(_Linear, x, weight, bias, residual, ACT_IDS[act] if not isinstance(act, int) else act, weight_kn,
                         float(dropout_p), float(alpha))


class _MLP(torch.autograd.Function):
    """y = dropout(act(x W1^T + b1) W2^T + b2) + residual.  The backward applies act'(pre-activation) to the second layer's
    dgrad output in one elementwise pass, which also accumulates the first layer's bias gradient into its flat slot."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, residual, act, weight_kn, dropout_p):
        x2 = _as2d(_bf16c(x))
        need = _grad_on and any(ctx.needs_input_grad)
        H = w1.shape[1] if weight_kn else w1.shape[0]
        N = w2.shape[1] if weight_kn else w2.shape[0]
        aux = torch.empty((x2.shape[0], H), device=x2.device, dtype=torch.bfloat16) if need else None
        h = L.gemm(x2, w1, b_mn=weight_kn, bias=b1, act=act, aux_out=aux)
        seed = next_seed() if dropout_p > 0 else 0
        res2 = _as2d(_bf16c(residual)) if residual is not None else None
        y = L.gemm(h, w2, b_mn=weight_kn, bias=b2, residual=res2, dropout_p=dropout_p, dropout_seed=seed,
                   dropout_seed_ptr=seed_counter(x2.device) if dropout_p > 0 else None)
        if need:
            ctx.save_for_backward(x2, aux, h)
        ctx.params = (w1, b1, w2, b2)
        ctx.meta = (act, weight_kn, dropout_p, seed, x.shape, residual.shape if residual is not None else None)
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        x2, aux, h = ctx.saved_tensors
        w1, b1, w2, b2 = ctx.params
        act, weight_kn, dropout_p, seed, xshape, res_shape = ctx.meta
        dy2 = _as2d(_bf16c(dy))
        d_res = dy.view(res_shape) if res_shape is not None and ctx.needs_input_grad[5] else None
        dz2 = L.dropout(dy2, dropout_p, seed, seed_ptr=seed_counter(dy2.device)) if dropout_p > 0 else dy2
        # (dZ2 W2) * act'(pre) in a separate pass: in the GEMM's epilogue (aux_in) the act' evaluation would sit on the
        # GEMM's critical path
        dh, b1_done = _act_bwd_with_bias_grad(L.gemm(dz2, w2, b_mn=not weight_kn), aux, act, b1)
        dw1 = dw2 = db1 = db2 = dx = None
        if w2.requires_grad:
            dw2 = _accum_grad_2d(w2, h, dz2, True, True) if weight_kn else _accum_grad_2d(w2, dz2, h, True, True)
        if b2 is not None and b2.requires_grad:
            db2 = _accum_bias_grad(b2, dz2)
        if ctx.needs_input_grad[0]:
            dx = L.gemm(dh, w1, b_mn=not weight_kn).view(xshape)
        if w1.requires_grad:
            dw1 = _accum_grad_2d(w1, x2, dh, True, True) if weight_kn else _accum_grad_2d(w1, dh, x2, True, True)
        if b1 is not None and b1.requires_grad and not b1_done:
            db1 = _accum_bias_grad(b1, dh)
        return dx, dw1, db1, dw2, db2, d_res, None, None, None


def mlp(x, w1, b1, w2, b2, *, act, residual=None, weight_kn=False, dropout_p=0.0):
    """Two-layer MLP block (timm Mlp / GPT2MLP / Perceiver FeedForward) on two fused-epilogue GEMMs."""
    return _apply(_MLP, x, w1, b1, w2, b2, residual, ACT_IDS[act] if not isinstance(act, int) else act, weight_kn,
                      float(dropout_p))


class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x2 = _as2d(_bf16c(x))
        need = _grad_on and any(ctx.needs_input_grad)
        y, mean, rstd = L.layernorm_fwd(x2, gamma, beta, eps, save_stats=need)
        if need:
            ctx.save_for_backward(x2, mean, rstd)
        ctx.gamma, ctx.beta = gamma, beta
        ctx.xshape = x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, mean, rstd = ctx.saved_tensors
        gamma, beta = ctx.gamma, ctx.beta
        dy2 = _as2d(_bf16c(dy))
        dg = db = None
        dg32 = db32 = None
        fused = False
        if gamma is not None and gamma.requires_grad:
            dg32 = getattr(gamma, "_dvla_grad32", None)
            db32 = getattr(beta, "_dvla_grad32", None) if beta is not None else None
            fused = dg32 is not None
            if not fused:
                dg32 = torch.zeros(x2.shape[1], device=x2.device, dtype=torch.float32)
                db32 = torch.zeros(x2.shape[1], device=x2.device, dtype=torch.float32) if beta is not None else None
        dx = L.layernorm_bwd(dy2, x2, gamma, mean, rstd, dg32, db32)
        if dg32 is not None and not fused:
            dg = dg32.to(torch.bfloat16)
            db = db32.to(torch.bfloat16) if db32 is not None else None
        return dx.view(ctx.xshape), dg, db, None


def layer_norm(x, gamma, beta, eps=1e-5):
    return _apply(_LayerNorm, x, gamma, beta, float(eps))


class _LayerNormFork(torch.autograd.Function):
    """(x, LN(x)) for pre-norm residual blocks `x + f(LN(x))`: the first output carries x into the residual add, so that
    BOTH gradients of x meet in this node and the LayerNorm-backward kernel emits their sum (dres) -- autograd would
    otherwise add them with a separate elementwise kernel per block."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x2 = _as2d(_bf16c(x))
        need = _grad_on and any(ctx.needs_input_grad)
        y, mean, rstd = L.layernorm_fwd(x2, gamma, beta, eps, save_stats=need)
        if need:
            ctx.save_for_backward(x2, mean, rstd)
        ctx.gamma, ctx.beta = gamma, beta
        ctx.xshape = x.shape
        return x.view_as(x), y.view(x.shape)

    @staticmethod
    def backward(ctx, dx_res, dy):
        x2, mean, rstd = ctx.saved_tensors
        gamma, beta = ctx.gamma, ctx.beta
        if dy is None:                      # LN output unused: only the pass-through gradient
            return dx_res, None, None, None
        dy2 = _as2d(_bf16c(dy))
        dres2 = _as2d(_bf16c(dx_res)) if dx_res is not None else None
        dg = db = dg32 = db32 = None
        fused = False
        if gamma is not None and gamma.requires_grad:
            dg32 = getattr(gamma, "_dvla_grad32", None)
            db32 = getattr(beta, "_dvla_grad32", None) if beta is not None else None
            fused = dg32 is not None
            if not fused:
                dg32 = torch.zeros(x2.shape[1], device=x2.device, dtype=torch.float32)
                db32 = torch.zeros(x2.shape[1], device=x2.device, dtype=torch.float32) if beta is not None else None
        dx = L.layernorm_bwd(dy2, x2, gamma, mean, rstd, dg32, db32, dres2)
        if dg32 is not None and not fused:
            dg = dg32.to(torch.bfloat16)
            db = db32.to(torch.bfloat16) if db32 is not None else None
        return dx.view(ctx.xshape), dg, db, None


def layer_norm_fork(x, gamma, beta, eps=1e-5):
    """-> (x for the residual branch, LayerNorm(x)); see _LayerNormFork."""
    return _apply(_LayerNormFork, x, gamma, beta, float(eps))


class AttnMask:
    """Bit-matrix visibility mask + per-tile flags, built once per mask (dreamvla_model.py:25-66 semantics:
    additive 0 -> visible, -inf -> hidden).  Shared across batch and heads."""

    @staticmethod
    def pack_bits(visible_bool: torch.Tensor) -> torch.Tensor:
        """[Lq, Lk] bool -> [Lq, ceil(Lk/32)] int32; bit (j % 32) of word (j // 32) set <=> pair (i, j) visible."""
        assert visible_bool.dim() == 2 and visible_bool.dtype == torch.bool
        Lq, Lk = visible_bool.shape
        words = (Lk + 31) // 32
        padded = torch.zeros(Lq, words * 32, dtype=torch.bool)
        padded[:, :Lk] = visible_bool.cpu()
        w = padded.view(Lq, words, 32).to(torch.int64)
        bits = (w << torch.arange(32, dtype=torch.int64)).sum(-1)
        return torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32)

    def __init__(self, visible_bool: torch.Tensor, device):
        self.Lq, self.Lk = visible_bool.shape
        self.bits = self.pack_bits(visible_bool).to(device).contiguous()
        self.flags = L.attn_mask_tiles(self.bits, self.Lq, self.Lk)

    @staticmethod
    def from_additive(mask_float: torch.Tensor, device):
        return AttnMask(mask_float == 0, device)

    @staticmethod
    def causal(n: int, device):
        return AttnMask(torch.ones(n, n, dtype=torch.bool).tril(), device)


class ObsDropMask(AttnMask):
    """AttnMask redrawn on the device: every draw() hides `count` of each timestep's n_obs observation columns from that
    timestep's action rows (the pretrain phase's per-forward drop, dreamvla_model.py:55-59), writing `bits` and `flags` in
    place.  Buffers are allocated once and nothing is read back, so a draw can be captured in a CUDA graph; the attention ops
    of a forward and its backward read the same buffers.  Draw rule: include/dvla.h dvla_attn_mask_obs_drop."""

    def __init__(self, base_visible: torch.Tensor, device, K: int, num_A: int, n_obs: int, n_act: int, count: int, seed: int):
        super().__init__(base_visible, device)
        self.base_bits = self.bits.clone()
        self.layout = (K, self.Lq // K, num_A, n_obs, n_act, count)
        self.seed = int(seed)

    def draw(self, seed_ptr: torch.Tensor):
        """Redraw under the effective seed `seed + *seed_ptr` (seed_ptr: device int64 counter, ops.seed_counter)."""
        if self.layout[3] > 0:          # no observation tokens: nothing to drop, the base mask stands
            L.attn_mask_obs_drop(self.base_bits, self.bits, self.flags, *self.layout, self.seed, seed_ptr)
        return self


class _CatBroadcast(torch.autograd.Function):
    """[n, a, C] per-sequence rows + [b, C] rows shared by every sequence -> [n, a + b, C]; the gradient of the shared rows
    is the sum over sequences (column-sum kernel over the [n, b*C] view of the incoming gradient)."""

    @staticmethod
    def forward(ctx, e, m):
        ctx.shapes = (e.shape, m.shape)
        return L.cat_broadcast(_bf16c(e), _bf16c(m))

    @staticmethod
    def backward(ctx, dy):
        (n, a, C), (b, _) = ctx.shapes
        dy = _bf16c(dy)
        de = dm = None
        if ctx.needs_input_grad[0]:
            de = dy[:, :a].contiguous()
        if ctx.needs_input_grad[1]:
            acc = torch.zeros(b * C, device=dy.device, dtype=torch.float32)
            L.colsum_accum(dy.view(n, (a + b) * C)[:, a * C:], acc)
            dm = acc.to(torch.bfloat16).view(b, C)
        return de, dm


def cat_broadcast(e, m):
    """torch.cat((e, m.expand(n, -1, -1)), dim=1) as one kernel each way (see _CatBroadcast)."""
    return _apply(_CatBroadcast, e, m)


class _Attention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale, mask, dropout_p, key_bias=None):
        need = _grad_on and any(ctx.needs_input_grad)
        seed = next_seed() if dropout_p > 0 else 0
        bits = mask.bits if mask is not None else None
        flags = mask.flags if mask is not None else None
        if mask is not None:
            assert mask.Lq == q.shape[1] and mask.Lk == k.shape[1], "mask shape mismatch"
        o, lse = L.attn_fwd(q, k, v, scale, bits, flags, dropout_p, seed, need_lse=need,
                            dropout_seed_ptr=seed_counter(q.device) if dropout_p > 0 else None, key_bias=key_bias)
        if need:
            ctx.save_for_backward(q, k, v, o, lse)
        ctx.meta = (scale, mask, dropout_p, seed, key_bias)
        return o

    @staticmethod
    def backward(ctx, d_o):
        q, k, v, o, lse = ctx.saved_tensors
        scale, mask, dropout_p, seed, key_bias = ctx.meta
        d_o = _bf16c(d_o)
        # if q, k, v are slices of one fused [B, L, 3, H, hd] buffer, produce the gradient in the same fused layout
        fused = (q.dim() == 4 and q._base is not None and q._base is k._base and q._base is v._base and
                 q._base.dim() == 5 and q._base.shape[2] == 3 and q._base.is_contiguous())
        if fused:
            dqkv = torch.empty_like(q._base)
            dq, dk, dv = dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2]
        else:
            dq = torch.empty(q.shape, device=q.device, dtype=torch.bfloat16)
            dk = torch.empty(k.shape, device=k.device, dtype=torch.bfloat16)
            dv = torch.empty(v.shape, device=v.device, dtype=torch.bfloat16)
        L.attn_bwd(q, k, v, o, d_o, lse, scale, dq, dk, dv, mask.bits if mask is not None else None,
                   mask.flags if mask is not None else None, dropout_p, seed,
                   dropout_seed_ptr=seed_counter(q.device) if dropout_p > 0 else None,
                   key_bias=key_bias)
        return dq, dk, dv, None, None, None, None


def attention(q, k, v, scale, mask: AttnMask | None = None, dropout_p: float = 0.0, key_bias=None):
    """q [B,Lq,H,hd], k/v [B,Lk,H,hd] (strided views allowed) -> [B,Lq,H,hd] contiguous.  hd = 64, or 96 on short
    sequences (Lq <= 32, Lk <= 64, no mask, no dropout).
    key_bias: optional fp32 [Lk] added to the scaled scores (log r = key counted r times); short sequences only."""
    return _apply(_Attention, q, k, v, float(scale), mask, float(dropout_p), key_bias)


class _FusedQKVAttention(torch.autograd.Function):
    """Self-attention on a fused qkv buffer [B, L, 3, H, hd]; the backward writes one fused dqkv buffer (no cat)."""

    @staticmethod
    def forward(ctx, qkv, scale, mask, dropout_p):
        need = _grad_on and any(ctx.needs_input_grad)
        seed = next_seed() if dropout_p > 0 else 0
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        o, lse = L.attn_fwd(q, k, v, scale, mask.bits if mask is not None else None,
                            mask.flags if mask is not None else None, dropout_p, seed, need_lse=need,
                            dropout_seed_ptr=seed_counter(qkv.device) if dropout_p > 0 else None)
        if need:
            ctx.save_for_backward(qkv, o, lse)
        ctx.meta = (scale, mask, dropout_p, seed)
        return o

    @staticmethod
    def backward(ctx, d_o):
        qkv, o, lse = ctx.saved_tensors
        scale, mask, dropout_p, seed = ctx.meta
        d_o = _bf16c(d_o)
        dqkv = torch.empty_like(qkv)
        L.attn_bwd(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], o, d_o, lse, scale, dqkv[:, :, 0], dqkv[:, :, 1],
                   dqkv[:, :, 2], mask.bits if mask is not None else None, mask.flags if mask is not None else None,
                   dropout_p, seed, dropout_seed_ptr=seed_counter(qkv.device) if dropout_p > 0 else None)
        return dqkv, None, None, None


def self_attention_fused(qkv, scale, mask: AttnMask | None = None, dropout_p: float = 0.0):
    """qkv [B, L, 3, H, hd] contiguous bf16 -> [B, L, H, hd]; hd = 64, or 96 on short sequences (see `attention`)."""
    assert qkv.dim() == 5 and qkv.shape[2] == 3 and qkv.shape[4] in (64, 96) and qkv.is_contiguous()
    return _apply(_FusedQKVAttention, qkv, float(scale), mask, float(dropout_p))


class _Dropout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p):
        seed = next_seed()
        ctx.meta = (p, seed, x.shape)
        return L.dropout(_as2d(_bf16c(x)), p, seed, seed_ptr=seed_counter(x.device)).view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        p, seed, shape = ctx.meta
        return L.dropout(_as2d(_bf16c(dy)), p, seed, seed_ptr=seed_counter(dy.device)).view(shape), None


def dropout(x, p: float, training: bool = True):
    if not training or p <= 0:
        return x
    return _apply(_Dropout, x, float(p))


# ----------------------------------------------------------------------------------------------------------------------
# fused losses: value is accumulated into a caller-provided fp32 scalar; gradient produced in the same pass
# ----------------------------------------------------------------------------------------------------------------------
class _LossBase(torch.autograd.Function):
    @staticmethod
    def backward(ctx, dloss):
        (dpred,) = ctx.saved_tensors
        # dpred already carries the loss weight; dloss is the upstream scalar (1/accum etc.)
        if ctx.unit_upstream:
            return (dpred.view(ctx.pshape),) + (None,) * ctx.nrest
        return ((dpred.float() * dloss).to(torch.bfloat16).view(ctx.pshape),) + (None,) * ctx.nrest


class _MSELoss(_LossBase):
    @staticmethod
    def forward(ctx, pred, label, row_mask, weight, unit_upstream):
        p2, l2 = _as2d(_bf16c(pred)), _as2d(_bf16c(label))
        loss = torch.zeros(1, device=pred.device, dtype=torch.float32)
        dpred = torch.empty_like(p2) if ctx.needs_input_grad[0] else None
        L.mse_loss(p2, l2, row_mask, weight, loss, dpred)
        if dpred is not None:
            ctx.save_for_backward(dpred)
        ctx.pshape, ctx.nrest, ctx.unit_upstream = pred.shape, 4, unit_upstream
        return loss[0]


def mse_loss(pred, label, row_mask=None, weight=1.0, unit_upstream=False):
    """weight * mean((pred*m - label*m)^2); row_mask fp32 [rows] of {0,1} (train_utils.py:325-337)."""
    return _MSELoss.apply(pred, label, row_mask, float(weight), unit_upstream)


class _CosineLoss(_LossBase):
    @staticmethod
    def forward(ctx, pred, label, weight, unit_upstream):
        p2, l2 = _as2d(_bf16c(pred)), _as2d(_bf16c(label))
        loss = torch.zeros(1, device=pred.device, dtype=torch.float32)
        dpred = torch.empty_like(p2) if ctx.needs_input_grad[0] else None
        L.cosine_loss(p2, l2, weight, loss, dpred)
        if dpred is not None:
            ctx.save_for_backward(dpred)
        ctx.pshape, ctx.nrest, ctx.unit_upstream = pred.shape, 3, unit_upstream
        return loss[0]


def cosine_loss(pred, label, weight=1.0, unit_upstream=False):
    """weight * mean(1 - cos(pred, label, dim=-1))  (train_utils.py:423-425)."""
    return _CosineLoss.apply(pred, label, float(weight), unit_upstream)


class _SiLogLoss(_LossBase):
    @staticmethod
    def forward(ctx, pred, label, lambd, weight, unit_upstream):
        p, l = _bf16c(pred), _bf16c(label)
        loss = torch.zeros(1, device=pred.device, dtype=torch.float32)
        dpred = torch.empty_like(p) if ctx.needs_input_grad[0] else None
        L.silog_loss(p, l, lambd, weight, loss, dpred)
        if dpred is not None:
            ctx.save_for_backward(dpred)
        ctx.pshape, ctx.nrest, ctx.unit_upstream = pred.shape, 4, unit_upstream
        return loss[0]


def silog_loss(pred, label, lambd=0.5, weight=1.0, unit_upstream=False):
    """Scale-invariant log loss (utils/sigloss.py:11-15); pred, label same shape (any)."""
    return _SiLogLoss.apply(pred, label, float(lambd), float(weight), unit_upstream)
