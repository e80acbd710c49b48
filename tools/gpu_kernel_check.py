"""Diagnostic sweep of every kernel in libdvla_sm90.so against plain PyTorch fp32 references ON THE GPU.

Usage (on an H100):  python tools/gpu_kernel_check.py <group> [--json out.json]
Groups run in separate processes (a trapped kernel poisons its CUDA context).  This is a development tool;
the graded parity tests are tests/test_*_gpu.py.
"""
from __future__ import annotations

import json
import math
import sys
import time

import numpy as np
import torch

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
from dreamvla_b200 import _lib as L  # noqa: E402

dev = "cuda"
RESULTS = []


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def report(name, err, tol, extra=""):
    ok = bool(err <= tol) and math.isfinite(err)
    RESULTS.append({"name": name, "err": err, "tol": tol, "ok": ok, "extra": extra})
    print(f"{'PASS' if ok else 'FAIL'} {name:58s} err={err:.3e} tol={tol:.1e} {extra}", flush=True)


def bench(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def act_ref(x, act):
    import torch.nn.functional as F
    if act == L.ACT_GELU_ERF: return F.gelu(x)
    if act == L.ACT_GELU_TANH: return F.gelu(x, approximate="tanh")
    if act == L.ACT_QUICK_GELU: return x * torch.sigmoid(1.702 * x)
    if act == L.ACT_RELU: return F.relu(x)
    if act == L.ACT_SILU: return F.silu(x)
    return x


def gemm_case(M, N, K, a_mn, b_mn, seed=0, timeit=False):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
    B = (torch.randn(N, K, generator=g) * 0.5).to(dev, torch.bfloat16)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    ref = A.float() @ B.float().t()
    out = L.gemm(a, b, a_mn=a_mn, b_mn=b_mn)
    torch.cuda.synchronize()
    extra = ""
    if timeit:
        ms = bench(lambda: L.gemm(a, b, a_mn=a_mn, b_mn=b_mn))
        extra = f"{ms*1e3:.1f}us {2*M*N*K/ms/1e9:.0f} TFLOP/s"
    report(f"gemm M{M} N{N} K{K} a_mn={int(a_mn)} b_mn={int(b_mn)}", rel(out, ref), 6e-3, extra)


def gemm_accum_case(M, N, K, seed=0, timeit=True):
    """weight-gradient form: G[M,N] += A[K,M]^T . B[K,N] (both operands MN-major), split-K eligible"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = (torch.randn(K, M, generator=g) * 0.5).to(dev, torch.bfloat16)
    b = (torch.randn(K, N, generator=g) * 0.5).to(dev, torch.bfloat16)
    G0 = (torch.randn(M, N, generator=g) * 4.0).to(dev, torch.bfloat16)
    ref = G0.float() + a.float().t() @ b.float()
    G = G0.clone()
    L.gemm(a, b, a_mn=True, b_mn=True, out=G, residual=G)
    torch.cuda.synchronize()
    extra = ""
    if timeit:
        scratch = torch.zeros_like(G)
        ms = bench(lambda: L.gemm(a, b, a_mn=True, b_mn=True, out=scratch, residual=scratch, alpha=1e-3))
        extra = f"{ms*1e3:.1f}us {2*M*N*K/ms/1e9:.0f} TFLOP/s"
    report(f"gemm accumulate (wgrad) M{M} N{N} K{K}", rel(G, ref), 6e-3, extra)


def group_gemm_splitk():
    gemm_accum_case(1024, 1024, 10320)
    gemm_accum_case(1024, 1024, 42400)
    gemm_accum_case(1024, 3072, 10320)
    gemm_accum_case(3072, 1024, 10320)
    gemm_accum_case(1024, 768, 10320)
    gemm_accum_case(768, 768, 31520)
    gemm_accum_case(768, 3072, 31520)
    gemm_accum_case(2304, 768, 31520)
    gemm_accum_case(520, 264, 4104)      # tails in M, N and K with splits
    gemm_accum_case(128, 136, 2048 + 8)


def group_gemm_basic():
    for a_mn in (False, True):
        for b_mn in (False, True):
            gemm_case(128, 128, 64, a_mn, b_mn)
            gemm_case(256, 512, 256, a_mn, b_mn)
            gemm_case(200, 264, 72, a_mn, b_mn)        # tails in M, N, K


def group_gemm_big():
    for a_mn in (False, True):
        for b_mn in (False, True):
            gemm_case(2580, 3072, 1024, a_mn, b_mn, timeit=True)
    gemm_case(2580, 1024, 4096, False, True, timeit=True)
    gemm_case(8200, 4096, 1024, False, False, timeit=True)
    gemm_case(7880, 2304, 768, False, False, timeit=True)
    gemm_case(3072, 1024, 2580, True, True, timeit=True)   # wgrad shape
    gemm_case(640, 3072, 768, False, False, timeit=True)
    gemm_case(8192, 8192, 8192, False, False, timeit=True)
    # cuBLAS for comparison
    for (M, N, K) in [(2580, 3072, 1024), (8200, 4096, 1024), (8192, 8192, 8192)]:
        A = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        B = torch.randn(N, K, device=dev, dtype=torch.bfloat16)
        ms = bench(lambda: torch.matmul(A, B.t()))
        print(f"INFO cublas M{M} N{N} K{K}: {ms*1e3:.1f}us {2*M*N*K/ms/1e9:.0f} TFLOP/s", flush=True)


def group_gemm_epilogue():
    g = torch.Generator(device="cpu").manual_seed(1)
    M, N, K = 300, 520, 256
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
    W = (torch.randn(N, K, generator=g) * 0.1).to(dev, torch.bfloat16)
    bias = torch.randn(N, generator=g).to(dev, torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(dev, torch.bfloat16)
    pre_ref = A.float() @ W.float().t() + bias.float()
    for act in (L.ACT_NONE, L.ACT_GELU_ERF, L.ACT_GELU_TANH, L.ACT_QUICK_GELU, L.ACT_RELU, L.ACT_SILU):
        aux = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        out = L.gemm(A, W, bias=bias, act=act, residual=res, aux_out=aux)
        report(f"gemm epi bias+act{act}+res", rel(out, act_ref(pre_ref, act) + res.float()), 6e-3)
        report(f"gemm epi aux_out act{act}", rel(aux, pre_ref), 6e-3)
        # dgrad through the activation: dX = (dY @ W) * act'(pre)   [here: reuse shapes: dY [M,K2] @ W2[K2->N]]
        pre = aux
        dy = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
        W2 = (torch.randn(K, N, generator=g) * 0.1).to(dev, torch.bfloat16)  # [K, N]: B n-major
        outg = L.gemm(dy, W2, b_mn=True, aux_in=pre, act=act)
        x = pre.float().requires_grad_(True)
        y = act_ref(x, act)
        gref = torch.autograd.grad(y, x, dy.float() @ W2.float())[0]
        report(f"gemm epi dact act{act}", rel(outg, gref), 8e-3)
    # fp32 output with accumulation into itself
    acc = torch.randn(M, N, device=dev, dtype=torch.float32)
    ref = acc + 0.5 * (A.float() @ W.float().t())
    L.gemm(A, W, out=acc, residual=acc, alpha=0.5)
    report("gemm epi fp32 accumulate alpha", rel(acc, ref), 1e-5)
    # bf16 accumulate in place
    accb = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
    refb = accb.float() + A.float() @ W.float().t()
    L.gemm(A, W, out=accb, residual=accb)
    report("gemm epi bf16 accumulate", rel(accb, refb), 6e-3)
    # dropout: statistics + exact mask agreement with dvla_dropout
    p = 0.1
    plain = L.gemm(A, W)
    dropped = L.gemm(A, W, dropout_p=p, dropout_seed=1234)
    again = L.dropout(plain, p, 1234)
    frac = (dropped == 0).float().mean().item()
    report("gemm epi dropout frac", abs(frac - p), 0.01, f"frac={frac:.4f}")
    report("gemm epi dropout == dropout kernel (values)", rel(dropped, again), 5e-3)
    report("gemm epi dropout == dropout kernel (mask)", ((dropped == 0) != (again == 0)).float().mean().item(), 1e-4)
    # tiny dims: K = 6 and 5 rows are not 16-byte multiples (SIMT kernel); N = 7 with 16-byte rows of A and B runs on the
    # wgmma kernel with the per-element epilogue (ldo = 7)
    for (M2, N2, K2, path) in [(20, 1024, 6, "simt"), (960, 7, 768, "wgmma direct"), (37, 13, 5, "simt")]:
        A2 = torch.randn(M2, K2, generator=g).to(dev, torch.bfloat16)
        W2 = torch.randn(N2, K2, generator=g).to(dev, torch.bfloat16)
        b2 = torch.randn(N2, generator=g).to(dev, torch.bfloat16)
        o2 = L.gemm(A2, W2, bias=b2)
        report(f"gemm {path} M{M2} N{N2} K{K2}", rel(o2, A2.float() @ W2.float().t() + b2.float()), 6e-3)
        # wgrad-like: dW[N2,K2] = dY^T X : a = dY [M2,N2] mn-major, b = X [M2,K2] mn-major
        dY = torch.randn(M2, N2, generator=g).to(dev, torch.bfloat16)
        o3 = L.gemm(dY, A2, a_mn=True, b_mn=True)
        report(f"gemm simt wgrad M{M2} N{N2} K{K2}", rel(o3, dY.float().t() @ A2.float()), 6e-3)


def group_norm():
    import torch.nn.functional as F
    g = torch.Generator(device="cpu").manual_seed(2)
    for (rows, D) in [(1000, 1024), (333, 768), (77, 512), (5, 384), (4099, 1024), (2600, 768), (3000, 512)]:     # >= 2048 rows: v2 kernel
        x = (torch.randn(rows, D, generator=g) * 2 + 0.5).to(dev, torch.bfloat16)
        gm = (1 + 0.1 * torch.randn(D, generator=g)).to(dev, torch.bfloat16)
        bt = (0.1 * torch.randn(D, generator=g)).to(dev, torch.bfloat16)
        for affine in (True, False):
            y, mean, rstd = L.layernorm_fwd(x, gm if affine else None, bt if affine else None, 1e-5)
            xr = x.float().requires_grad_(True)
            gr = gm.float().requires_grad_(True)
            br = bt.float().requires_grad_(True)
            yr = F.layer_norm(xr, (D,), gr if affine else None, br if affine else None, 1e-5)
            report(f"layernorm fwd {rows}x{D} affine={int(affine)}", rel(y, yr), 5e-3)
            dy = torch.randn(rows, D, generator=g).to(dev, torch.bfloat16)
            dg = torch.zeros(D, device=dev) if affine else None
            db = torch.zeros(D, device=dev) if affine else None
            dx = L.layernorm_bwd(dy, x, gm if affine else None, mean, rstd, dg, db)
            yr.backward(dy.float())
            report(f"layernorm bwd dx {rows}x{D} affine={int(affine)}", rel(dx, xr.grad), 8e-3)
            dres = torch.randn(rows, D, generator=g).to(dev, torch.bfloat16)       # + residual-branch gradient (fork)
            dx2 = L.layernorm_bwd(dy, x, gm if affine else None, mean, rstd, None, None, dres)
            report(f"layernorm bwd dx+dres {rows}x{D} affine={int(affine)}", rel(dx2, xr.grad + dres.float()), 8e-3)
            if affine:
                report(f"layernorm bwd dgamma {rows}x{D}", rel(dg, gr.grad), 8e-3)
                report(f"layernorm bwd dbeta {rows}x{D}", rel(db, br.grad), 8e-3)
    # the fused form the blocks use (dres + dgamma/dbeta in one launch), timed at the decoder and backbone sizes
    for rows in (42400, 10320):
        x = torch.randn(rows, 1024, generator=g).to(dev, torch.bfloat16)
        gm = torch.ones(1024, device=dev, dtype=torch.bfloat16)
        y, mean, rstd = L.layernorm_fwd(x, gm, gm, 1e-5)
        dy = torch.randn(rows, 1024, generator=g).to(dev, torch.bfloat16)
        dres = torch.randn(rows, 1024, generator=g).to(dev, torch.bfloat16)
        dg, db = torch.zeros(1024, device=dev), torch.zeros(1024, device=dev)
        dx = L.layernorm_bwd(dy, x, gm, mean, rstd, dg, db, dres)
        xr = x.float().requires_grad_(True)
        gr = gm.float().requires_grad_(True)
        br = gm.float().requires_grad_(True)
        F.layer_norm(xr, (1024,), gr, br, 1e-5).backward(dy.float())
        e_dx, e_dg, e_db = rel(dx, xr.grad + dres.float()), rel(dg, gr.grad), rel(db, br.grad)
        dg2, db2 = torch.zeros(1024, device=dev), torch.zeros(1024, device=dev)
        ms = bench(lambda: L.layernorm_bwd(dy, x, gm, mean, rstd, dg2, db2, dres))
        gbs = rows * 1024 * 2 * 4 / ms / 1e6                       # x, dy, dres read + dx written
        report(f"layernorm bwd fused dx+dres {rows}x1024", e_dx, 8e-3, f"{ms*1e3:.1f}us {gbs:.0f} GB/s")
        report(f"layernorm bwd fused dgamma {rows}x1024", e_dg, 8e-3)
        report(f"layernorm bwd fused dbeta {rows}x1024", e_db, 8e-3)
    x = torch.randn(2580, 3072, generator=g).to(dev, torch.bfloat16)
    out = torch.zeros(3072, device=dev)
    L.colsum_accum(x, out)
    report("colsum 2580x3072", rel(out, x.float().sum(0)), 1e-4)
    x = torch.randn(37, 13, generator=g).to(dev, torch.bfloat16)
    out = torch.zeros(13, device=dev)
    L.colsum_accum(x, out)
    report("colsum 37x13 (scalar path)", rel(out, x.float().sum(0)), 1e-4)
    dst = torch.randn(1000, generator=g).to(dev, torch.bfloat16)
    src = torch.randn(1000, generator=g).to(dev)
    ref = dst.float() + src
    L.accum_fp32_into_bf16(src, dst)
    report("accum_fp32_into_bf16", rel(dst, ref), 5e-3)


def attn_ref(q, k, v, scale, mask_bool):
    # q [B,Lq,H,64] ... -> o [B,Lq,H,64]; fp32
    qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
    s = (qf @ kf.transpose(-1, -2)) * scale
    if mask_bool is not None:
        s = s.masked_fill(~mask_bool, float("-inf"))
    p = s.softmax(-1)
    return (p @ vf).permute(0, 2, 1, 3)


def pack_mask(mask_bool):
    Lq, Lk = mask_bool.shape
    words = (Lk + 31) // 32
    padded = torch.zeros(Lq, words * 32, dtype=torch.bool)
    padded[:, :Lk] = mask_bool.cpu()
    w = padded.view(Lq, words, 32).to(torch.int64)
    bits = (w << torch.arange(32, dtype=torch.int64)).sum(-1)
    bits = torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32)
    return bits.to(dev)


def attn_case(B, H, Lq, Lk, masked, fused_qkv=False, seed=3, timeit=False, ramp=0.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if fused_qkv:
        assert Lq == Lk
        qkv = torch.randn(B, Lq, 3, H, 64, generator=g).to(dev, torch.bfloat16)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    else:
        q = torch.randn(B, Lq, H, 64, generator=g).to(dev, torch.bfloat16)
        k = torch.randn(B, Lk, H, 64, generator=g).to(dev, torch.bfloat16)
        v = torch.randn(B, Lk, H, 64, generator=g).to(dev, torch.bfloat16)
        if ramp:      # key norms grow along the sequence: the running row max keeps rising (online-softmax rescale path)
            k = (k.float() * (1.0 + ramp * torch.arange(Lk, device=dev).view(1, Lk, 1, 1) / Lk)).to(torch.bfloat16)
            q = (q.float() * 2.0).to(torch.bfloat16)
    mask_bool = bits = flags = None
    if masked:
        mask_bool = torch.rand(Lq, Lk, generator=g) < 0.3
        mask_bool[:, 0] = True                       # no fully-masked rows
        if Lk > 130:
            mask_bool[: Lq // 2, 64:128] = False     # a fully masked tile
            mask_bool[Lq // 2:, 64:128] = True       # a fully visible one (if Lq//2 is tile aligned)
        bits = pack_mask(mask_bool)
        flags = L.attn_mask_tiles(bits, Lq, Lk)
        mask_bool = mask_bool.to(dev)
    scale = 0.125
    o, lse = L.attn_fwd(q, k, v, scale, bits, flags)
    qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    oref = attn_ref(qr, kr, vr, scale, mask_bool)
    tag = f"attn B{B} H{H} Lq{Lq} Lk{Lk} mask={int(masked)} fused={int(fused_qkv)}" + (f" ramp={ramp}" if ramp else "")
    extra = ""
    if timeit:
        ms = bench(lambda: L.attn_fwd(q, k, v, scale, bits, flags))
        extra = f"fwd {ms*1e3:.1f}us"
    report(tag + " fwd", rel(o, oref), 6e-3, extra)
    d_o = torch.randn(B, Lq, H, 64, generator=g).to(dev, torch.bfloat16)
    if fused_qkv:
        dqkv = torch.empty_like(qkv)
        dq, dk, dv = dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2]
    else:
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    L.attn_bwd(q, k, v, o, d_o, lse, scale, dq, dk, dv, bits, flags)
    oref.backward(d_o.float())
    if timeit:
        ms = bench(lambda: L.attn_bwd(q, k, v, o, d_o, lse, scale, dq, dk, dv, bits, flags))
        extra = f"bwd {ms*1e3:.1f}us"
    report(tag + " dq", rel(dq, qr.grad), 1e-2, extra)
    report(tag + " dk", rel(dk, kr.grad), 1e-2)
    report(tag + " dv", rel(dv, vr.grad), 1e-2)


def group_attn():
    attn_case(1, 1, 128, 128, False)
    attn_case(1, 2, 130, 257, False)
    attn_case(2, 2, 300, 140, True)
    attn_case(1, 1, 64, 64, False)
    attn_case(2, 3, 197, 197, False, fused_qkv=True)
    attn_case(2, 2, 16, 212, False)
    attn_case(1, 2, 6, 6, False)
    attn_case(5, 12, 6, 6, False, fused_qkv=True)              # DiT block (SIMT row kernels, attention_small.cu)
    attn_case(3, 2, 10, 265, False)                            # identical-mask-row decoder form
    attn_case(2, 3, 32, 40, False)
    attn_case(2, 2, 33, 40, False)                             # just above the short-query limit: mma.sync kernels
    attn_case(640, 12, 6, 6, False, fused_qkv=True, timeit=True)
    attn_case(160, 8, 16, 212, False, timeit=True)
    attn_case(320, 16, 10, 265, False, timeit=True)
    attn_case(1, 2, 265, 265, True)
    attn_case(1, 2, 258, 258, True, fused_qkv=True)
    attn_case(1, 2, 300, 520, False, ramp=6.0)
    attn_case(2, 2, 515, 700, True, ramp=4.0)
    attn_case(2, 16, 1290, 1290, True, fused_qkv=True, timeit=True)
    attn_case(40, 12, 197, 197, False, fused_qkv=True, timeit=True)
    attn_case(40, 16, 265, 265, False, fused_qkv=True, timeit=True)
    # key_bias = log(r): the last key counted r times == attention over r explicit copies of it (identical-mask-row decoders)
    g = torch.Generator(device="cpu").manual_seed(21)
    Bq, Hq, Lx, rep = 3, 2, 10, 256
    q = torch.randn(Bq, Lx, Hq, 64, generator=g).to(dev, torch.bfloat16)
    k = torch.randn(Bq, Lx, Hq, 64, generator=g).to(dev, torch.bfloat16)
    v = torch.randn(Bq, Lx, Hq, 64, generator=g).to(dev, torch.bfloat16)
    bias = torch.zeros(Lx, device=dev, dtype=torch.float32)
    bias[-1] = float(np.log(rep))
    o, lse = L.attn_fwd(q, k, v, 0.125, key_bias=bias)
    qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    kx = torch.cat((kr[:, :-1], kr[:, -1:].expand(-1, rep, -1, -1)), dim=1)
    vx = torch.cat((vr[:, :-1], vr[:, -1:].expand(-1, rep, -1, -1)), dim=1)
    oref = attn_ref(qr, kx, vx, 0.125, None)
    report("attn key_bias=log(256) fwd vs 256 explicit copies", rel(o, oref), 6e-3)
    d_o = torch.randn(Bq, Lx, Hq, 64, generator=g).to(dev, torch.bfloat16)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    L.attn_bwd(q, k, v, o, d_o, lse, 0.125, dq, dk, dv, key_bias=bias)
    oref.backward(d_o.float())
    # the 256-fold key takes ~all of the probability mass: dS = P (dP - delta) is a difference of nearly equal numbers and
    # delta = rowsum(dO * O) is formed from the bf16-ROUNDED output (FlashAttention-2 backward), hence the wider bar
    report("attn key_bias dq", rel(dq, qr.grad), 3e-2)
    report("attn key_bias dk (copies summed)", rel(dk, kr.grad), 3e-2)
    report("attn key_bias dv (copies summed)", rel(dv, vr.grad), 1e-2)
    # cat_broadcast fwd / bwd
    e = torch.randn(7, 9, 3072, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    m = torch.randn(196, 3072, generator=g).to(dev, torch.bfloat16).requires_grad_(True)
    from dreamvla_b200 import ops as _ops
    y = _ops.cat_broadcast(e, m)
    yref = torch.cat((e, m.unsqueeze(0).expand(7, -1, -1)), dim=1)
    report("cat_broadcast fwd (exact)", 0.0 if torch.equal(y, yref) else 1.0, 0.5)
    gy = torch.randn(7, 205, 3072, generator=g).to(dev, torch.bfloat16)
    y.backward(gy)
    report("cat_broadcast d(e) (exact)", 0.0 if torch.equal(e.grad, gy[:, :9]) else 1.0, 0.5)
    report("cat_broadcast d(m) = sum over sequences", rel(m.grad, gy[:, 9:].float().sum(0)), 5e-3)
    # dropout: statistical check (mean preserved) + fwd/bwd consistency via finite structure
    g = torch.Generator(device="cpu").manual_seed(5)
    q = torch.randn(2, 128, 4, 64, generator=g).to(dev, torch.bfloat16)
    k = torch.randn(2, 128, 4, 64, generator=g).to(dev, torch.bfloat16)
    v = torch.ones(2, 128, 4, 64, device=dev, dtype=torch.bfloat16)
    o, lse = L.attn_fwd(q, k, v, 0.125, dropout_p=0.25, dropout_seed=77)
    # with V == 1, o = sum_j keep_ij p_ij / (1-p): mean over i should be ~1
    report("attn dropout mean", abs(o.float().mean().item() - 1.0), 0.02, f"mean={o.float().mean().item():.4f}")
    o2, _ = L.attn_fwd(q, k, v, 0.125, dropout_p=0.25, dropout_seed=77)
    report("attn dropout deterministic", rel(o2, o), 1e-7)
    # backward with dropout: dV = P_drop^T dO. With dO = 1, dV[j,:] = sum_i P_drop[i,j]; sum_j dV[j,0] = sum_i o[i,0]
    d_o = torch.ones_like(o)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    L.attn_bwd(q, k, v, o, d_o, lse, 0.125, dq, dk, dv, dropout_p=0.25, dropout_seed=77)
    lhs = dv.float()[..., 0].sum(1)   # [B,H]
    rhs = o.float()[..., 0].sum(1)
    report("attn dropout bwd mask == fwd mask", rel(lhs, rhs), 5e-3)


def group_attn_perf():
    """fwd / bwd timings on the path's real attention shapes at per-GPU batch 8 (S = 10), real GPT-2 block mask"""
    from dreamvla_b200 import ops
    from dreamvla_b200.models.dreamvla_model import generate_attention_mask
    g = torch.Generator(device="cpu").manual_seed(11)

    def run(tag, B, H, L, mask=None, p=0.0):
        qkv = torch.randn(B, L, 3, H, 64, generator=g).to(dev, torch.bfloat16)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        bits = flags = None
        if mask is not None:
            bits, flags = mask.bits, mask.flags
        o, lse = L_.attn_fwd(q, k, v, 0.125, bits, flags, dropout_p=p, dropout_seed=5)
        d_o = torch.randn(B, L, H, 64, generator=g).to(dev, torch.bfloat16)
        dqkv = torch.empty_like(qkv)
        f = bench(lambda: L_.attn_fwd(q, k, v, 0.125, bits, flags, dropout_p=p, dropout_seed=5))
        bw = bench(lambda: L_.attn_bwd(q, k, v, o, d_o, lse, 0.125, dqkv[:, :, 0], dqkv[:, :, 1], dqkv[:, :, 2], bits, flags,
                                       dropout_p=p, dropout_seed=5))
        vis = float(L * L) if mask is None else float(mask.visible)
        gf = 4 * 64 * vis * B * H / 1e9
        print(f"INFO attn_perf {tag:28s} fwd {f*1e3:7.1f} us ({gf/f:6.0f} TF/s)  bwd {bw*1e3:7.1f} us ({2.5*gf/bw:6.0f} TF/s)", flush=True)

    L_ = L
    run("vit B160 H12 L197", 160, 12, 197)
    run("decoder B160 H16 L265", 160, 16, 265)
    run("decoder B160 H16 L205", 160, 16, 205)
    add = generate_attention_mask(K=10, num_A=36, num_B=93, atten_goal=0, atten_goal_state=False, atten_only_obs=False,
                                  attn_robot_proprio_state=False, mask_l_obs_ratio=0.0, num_obs_token=90, action_pred_steps=3)
    mb = (add == 0)
    if mb is not None:
        am = ops.AttnMask(mb, dev)
        am.visible = int(mb.sum().item())
        run("gpt2 B8 H16 L1290 mask", 8, 16, mb.shape[0], am)
        run("gpt2 B8 H16 L1290 mask drop", 8, 16, mb.shape[0], am, p=0.1)
    # grouped token order [A | queries | action]: every attendable key of the A / query rows sits in the first 36*S rows, so
    # the main call is (Lq = 1260 rows) x (Lk = 360 keys) with a dense step-causal mask, plus a 30-row call for the action rows
    S, n_a, n_q, n_act = 10, 36, 90, 3
    step_a = torch.arange(S).repeat_interleave(n_a)
    step_q = torch.arange(S).repeat_interleave(n_q)
    rows_step = torch.cat((step_a, step_q))
    mb_main = rows_step[:, None] >= step_a[None, :]                                    # [1260, 360]
    step_act = torch.arange(S).repeat_interleave(n_act)
    mb_act = torch.cat((step_act[:, None] >= step_a[None, :], step_act[:, None] == step_q[None, :]), dim=1)   # [30, 1260]
    am_main, am_act = ops.AttnMask(mb_main, dev), ops.AttnMask(mb_act, dev)
    for p_drop in (0.0, 0.1):
        B, H, Lt = 8, 16, S * (n_a + n_q + n_act)
        qkv = torch.randn(B, Lt, 3, H, 64, generator=g).to(dev, torch.bfloat16)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        n_main, n_ka = S * (n_a + n_q), S * n_a
        d_o = torch.randn(B, Lt, H, 64, generator=g).to(dev, torch.bfloat16)
        dqkv = torch.empty_like(qkv)
        dk_act, dv_act = torch.empty(B, n_main, H, 64, device=dev, dtype=torch.bfloat16), torch.empty(B, n_main, H, 64, device=dev, dtype=torch.bfloat16)

        def fwd():
            o1, l1 = L_.attn_fwd(q[:, :n_main], k[:, :n_ka], v[:, :n_ka], 0.125, am_main.bits, am_main.flags, dropout_p=p_drop, dropout_seed=5)
            o2, l2 = L_.attn_fwd(q[:, n_main:], k[:, :n_main], v[:, :n_main], 0.125, am_act.bits, am_act.flags, dropout_p=p_drop, dropout_seed=6)
            return o1, l1, o2, l2
        o1, l1, o2, l2 = fwd()

        def bwd():
            L_.attn_bwd(q[:, :n_main], k[:, :n_ka], v[:, :n_ka], o1, d_o[:, :n_main], l1, 0.125, dqkv[:, :n_main, 0], dqkv[:, :n_ka, 1],
                        dqkv[:, :n_ka, 2], am_main.bits, am_main.flags, dropout_p=p_drop, dropout_seed=5)
            L_.attn_bwd(q[:, n_main:], k[:, :n_main], v[:, :n_main], o2, d_o[:, n_main:], l2, 0.125, dqkv[:, n_main:, 0], dk_act, dv_act,
                        am_act.bits, am_act.flags, dropout_p=p_drop, dropout_seed=6)
        f, bw = bench(fwd), bench(bwd)
        print(f"INFO attn_perf gpt2 GROUPED main 1260x360 + act 30x1260, drop={p_drop}: fwd {f*1e3:7.1f} us  bwd {bw*1e3:7.1f} us", flush=True)
    report("attn_perf ran", 0.0, 1.0)


def group_loss():
    import torch.nn.functional as F
    g = torch.Generator(device="cpu").manual_seed(4)
    rows, Cc = 4000, 768
    pred = torch.randn(rows, Cc, generator=g).to(dev, torch.bfloat16)
    label = torch.randn(rows, Cc, generator=g).to(dev, torch.bfloat16)
    mask = (torch.rand(rows, generator=g) < 0.5).float().to(dev)
    for m in (None, mask):
        loss = torch.zeros(1, device=dev)
        dp = torch.empty_like(pred)
        L.mse_loss(pred, label, m, 0.1, loss, dp)
        pr = pred.float().requires_grad_(True)
        mm = 1.0 if m is None else m[:, None]
        lr_ = 0.1 * F.mse_loss(pr * mm, label.float() * mm)
        lr_.backward()
        report(f"mse loss mask={m is not None}", abs(loss.item() - lr_.item()) / abs(lr_.item()), 1e-4)
        report(f"mse dpred mask={m is not None}", rel(dp, pr.grad), 8e-3)
    loss = torch.zeros(1, device=dev)
    dp = torch.empty_like(pred)
    L.cosine_loss(pred, label, 0.01, loss, dp)
    pr = pred.float().requires_grad_(True)
    lr_ = 0.01 * (1 - F.cosine_similarity(pr, label.float(), dim=-1)).mean()
    lr_.backward()
    report("cosine loss", abs(loss.item() - lr_.item()) / abs(lr_.item()), 1e-4)
    report("cosine dpred", rel(dp, pr.grad), 8e-3)
    n = 20 * 224 * 224
    p = (torch.rand(n, generator=g) * 3 + 0.05).to(dev, torch.bfloat16)
    t = (torch.rand(n, generator=g) * 5 + 0.1).to(dev, torch.bfloat16)
    loss = torch.zeros(1, device=dev)
    dp = torch.empty_like(p)
    L.silog_loss(p, t, 0.5, 0.001, loss, dp)
    pr = p.float().requires_grad_(True)
    d = torch.log(t.float() + 1e-6) - torch.log(pr + 1e-6)
    lr_ = 0.001 * torch.sqrt((d ** 2).mean() - 0.5 * d.mean() ** 2)
    lr_.backward()
    report("silog loss", abs(loss.item() - lr_.item()) / abs(lr_.item()), 1e-3)
    report("silog dpred", rel(dp, pr.grad), 8e-3)
    # optimizer
    n = 1_000_003 + 5
    n = (n // 8) * 8 + 8
    P = torch.randn(n, generator=g).to(dev, torch.bfloat16)
    G = (torch.randn(n, generator=g) * 0.01).to(dev, torch.bfloat16)
    ss = torch.zeros(1, device=dev)
    L.sumsq(G, ss)
    report("sumsq", abs(ss.item() - (G.float() ** 2).sum().item()) / (G.float() ** 2).sum().item(), 1e-4)
    pref = P.float().clone().requires_grad_(True)
    opt = torch.optim.AdamW([pref], lr=1e-3, weight_decay=1e-2, betas=(0.9, 0.999), eps=1e-8)
    m = torch.zeros(n, device=dev)
    v = torch.zeros(n, device=dev)
    lr_t = torch.tensor([1e-3], device=dev)
    step_t = torch.zeros(1, device=dev)
    Pc = P.clone()
    for it in range(3):
        Gi = (G.float() * (it + 1)).to(torch.bfloat16)
        pref.grad = Gi.float().clone()
        torch.nn.utils.clip_grad_norm_([pref], 0.1)
        opt.step()
        ss.zero_()
        L.sumsq(Gi, ss)
        step_t += 1
        Gw = Gi.clone()
        L.adamw(Pc, Gw, m, v, sumsq_t=ss, lr_t=lr_t, step_t=step_t, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2,
                max_norm=0.1, zero_grad=True)
        assert Gw.abs().max().item() == 0
    report("adamw 3 steps (bf16 param rounding)", rel(Pc, pref.detach()), 8e-3)
    # fp32 master weights: the same 3 steps on fp32 parameters, the bf16 working copy rounded from the master
    P32 = P.float()
    pref = P32.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pref], lr=1e-3, weight_decay=1e-2, betas=(0.9, 0.999), eps=1e-8)
    m.zero_()
    v.zero_()
    step_t.zero_()
    Pw = torch.empty_like(P)
    for it in range(3):
        Gi = (G.float() * (it + 1)).to(torch.bfloat16)
        pref.grad = Gi.float().clone()
        torch.nn.utils.clip_grad_norm_([pref], 0.1)
        opt.step()
        ss.zero_()
        L.sumsq(Gi, ss)
        step_t += 1
        Gw = Gi.clone()
        L.adamw_master(P32, Pw, Gw, m, v, sumsq_t=ss, lr_t=lr_t, step_t=step_t, beta1=0.9, beta2=0.999, eps=1e-8,
                       weight_decay=1e-2, max_norm=0.1, zero_grad=True)
        assert Gw.abs().max().item() == 0
        assert torch.equal(Pw, P32.to(torch.bfloat16))
    report("adamw_master 3 steps (fp32 update)", rel(P32 - P.float(), pref.detach() - P.float()), 1e-5)
    _check_sumsq_deterministic()


def _check_sumsq_deterministic():
    """the gradient norm feeds every replica's clip factor: same buffer -> same bits, whatever the block scheduling"""
    g = torch.Generator(device="cpu").manual_seed(12)
    x = torch.randn(5_000_003, generator=g).to(dev, torch.bfloat16)[:5_000_000 - 8]
    outs = []
    for _ in range(5):
        o = torch.zeros(1, device=dev, dtype=torch.float32)
        L.sumsq(x, o)
        outs.append(o.clone())
    ref = (x.double() ** 2).sum()
    report("sumsq vs fp64", abs(float(outs[0]) - float(ref)) / float(ref), 1e-5)
    report("sumsq bit-reproducible", 0.0 if all(torch.equal(outs[0], o) for o in outs) else 1.0, 0.5)


def group_act_bwd_colsum():
    """dx = dy * act'(pre) (dvla_act_bwd) for every activation, and with the column sums of dx accumulated in the same pass
    (dvla_act_bwd_colsum)."""
    g = torch.Generator().manual_seed(11)
    for act in (L.ACT_NONE, L.ACT_GELU_ERF, L.ACT_GELU_TANH, L.ACT_QUICK_GELU, L.ACT_RELU, L.ACT_SILU):
        dy = (torch.randn(300, 256, generator=g) * 0.5).to(dev, torch.bfloat16)
        db = L.act_bwd(dy, dy, act)
        x2 = dy.float().requires_grad_(True)
        gref2 = torch.autograd.grad(act_ref(x2, act), x2, dy.float())[0]
        report(f"act_bwd act{act}", rel(db, gref2), 8e-3)
    for (rows, N, act) in [(777, 4096, L.ACT_GELU_ERF), (2600, 3072, L.ACT_GELU_TANH), (33, 264, L.ACT_SILU), (5, 4096, L.ACT_RELU),
                           (10320, 4096, L.ACT_GELU_TANH), (42400, 4096, L.ACT_GELU_ERF)]:
        dy = (torch.randn(rows, N, generator=g) * 0.5).to(dev, torch.bfloat16)
        pre = torch.randn(rows, N, generator=g).to(dev, torch.bfloat16)
        acc0 = torch.randn(N, generator=g).to(dev)
        acc = acc0.clone()
        dx = L.act_bwd(dy, pre, act, colsum_out=acc)
        x = pre.float().requires_grad_(True)
        gref = torch.autograd.grad(act_ref(x, act), x, dy.float())[0]
        report(f"act_bwd_colsum dx {rows}x{N} act{act}", rel(dx, gref), 8e-3)
        report(f"act_bwd_colsum sum {rows}x{N} act{act}", rel(acc - acc0, gref.sum(0)), 2e-3)
        plain = L.act_bwd(dy, pre, act)
        report(f"act_bwd_colsum dx == act_bwd {rows}x{N}", float((dx.float() - plain.float()).abs().max()), 0.0)
        if rows >= 10000:
            t_f = bench(lambda: L.act_bwd(dy, pre, act, colsum_out=acc))
            t_a = bench(lambda: L.act_bwd(dy, pre, act))
            t_c = bench(lambda: L.colsum_accum(plain, acc))
            by = rows * N * 6
            print(f"     fused {t_f*1e3:.1f} us ({by/t_f/1e6:.0f} GB/s)  vs  act_bwd {t_a*1e3:.1f} us + colsum {t_c*1e3:.1f} us", flush=True)


def group_gemm_tail():
    """K-split tail of the persistent GEMMs (partial last wave cut along K, fp32 reduction through the workspace):
    results against fp32 torch for every epilogue, repeated launches (self-cleaning workspace), timing of the step's shapes."""
    g = torch.Generator(device="cpu").manual_seed(5)
    for (M, N, K, b_mn) in [(10320, 1024, 4096, False), (10320, 1024, 4096, True), (10320, 1024, 3072, False),
                            (10320, 1024, 1024, True), (2580, 1024, 4096, False), (1300, 512, 2048, False),
                            (5000, 1000, 1536, True), (31520, 768, 3072, False)]:
        A = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
        W = (torch.randn(N, K, generator=g) * 0.05).to(dev, torch.bfloat16)
        w = W.t().contiguous() if b_mn else W
        bias = torch.randn(N, generator=g).to(dev, torch.bfloat16)
        res = torch.randn(M, N, generator=g).to(dev, torch.bfloat16)
        ref = A.float() @ W.float().t()
        out = L.gemm(A, w, b_mn=b_mn)
        report(f"gemm tail plain M{M} N{N} K{K} b_mn={int(b_mn)}", rel(out, ref), 6e-3)
        out2 = L.gemm(A, w, b_mn=b_mn)
        report(f"gemm tail repeat == first M{M} N{N} K{K}", 0.0 if torch.equal(out, out2) else 1.0, 0.0)   # fixed-order sum
        aux = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        out = L.gemm(A, w, b_mn=b_mn, bias=bias, act=L.ACT_GELU_TANH, residual=res, aux_out=aux)
        pre = ref + bias.float()
        report(f"gemm tail bias+gelu+res M{M} N{N} K{K}", rel(out, act_ref(pre, L.ACT_GELU_TANH) + res.float()), 6e-3)
        report(f"gemm tail aux_out M{M} N{N} K{K}", rel(aux, pre), 6e-3)
        ws = L.gemm_workspace(A.device)
        report(f"gemm tail counters left zero M{M} N{N} K{K}", float(ws[:65536].view(torch.int32).abs().max()), 0.0)
        ms = bench(lambda: L.gemm(A, w, b_mn=b_mn, bias=bias, residual=res))
        print(f"     M{M} N{N} K{K} b_mn={int(b_mn)} bias+res: {ms*1e3:.1f} us {2*M*N*K/ms/1e9:.0f} TFLOP/s", flush=True)
    # dropout epilogue: same mask as the stand-alone kernel
    M, N, K = 10320, 1024, 4096
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev, torch.bfloat16)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dev, torch.bfloat16)
    plain = L.gemm(A, W)
    dropped = L.gemm(A, W, dropout_p=0.1, dropout_seed=77)
    want = L.dropout(plain, 0.1, 77)
    report("gemm tail dropout epilogue == dropout(plain)", rel(dropped, want), 4e-3)


GROUPS = {"gemm_basic": group_gemm_basic, "gemm_splitk": group_gemm_splitk, "gemm_big": group_gemm_big, "gemm_epilogue": group_gemm_epilogue,
          "norm": group_norm, "attn": group_attn, "attn_perf": group_attn_perf, "loss": group_loss, "act_bwd_colsum": group_act_bwd_colsum, "gemm_tail": group_gemm_tail}

if __name__ == "__main__":
    grp = sys.argv[1]
    t0 = time.time()
    try:
        GROUPS[grp]()
    except Exception as e:  # noqa: BLE001
        import traceback
        traceback.print_exc()
        RESULTS.append({"name": f"{grp} EXCEPTION", "err": float("nan"), "tol": 0, "ok": False, "extra": repr(e)[:300]})
        print(f"FAIL {grp} EXCEPTION {e!r}", flush=True)
    torch.cuda.synchronize() if torch.cuda.is_available() else None
    nfail = sum(not r["ok"] for r in RESULTS)
    print(f"GROUP {grp}: {len(RESULTS) - nfail} pass, {nfail} fail, {time.time() - t0:.1f}s", flush=True)
    if "--json" in sys.argv:
        with open(sys.argv[sys.argv.index("--json") + 1], "w") as f:
            json.dump(RESULTS, f, indent=1)
    sys.exit(1 if nfail else 0)
