"""One table of dvla_gemm cases: every kernel path of the dispatcher crossed with the operand majornesses and epilogue
recipes, at the shapes where tiling goes wrong, with distinct row strides and element offsets for every matrix.

The CPU test (tests/test_gemm_plan_cpu.py) plans every case with fake pointers that carry its alignment and checks the
declared path at 132 and 114 SMs (H100 SXM and PCIe); the GPU test (tests/test_gemm_paths_gpu.py) runs every case against
an fp64 reference with guard bands around each output.

Paths (`dvla_gemm_plan` plus the staging rule of `dvla_gemm`, see `staging`):
  simt_thread          kernel 0: A or B not TMA-addressable, short contraction or large output
  simt_warp            kernel 1: A or B not TMA-addressable, K >= 128 and M * ceil(N/8) <= 65536
  wgmma_staged         kernel 2, whole tiles, smem-staged epilogue (bf16 out, 16-B aligned, N % 8 == 0)
  wgmma_direct_vec     kernel 2, per-8-column epilogue with 16-B vectors: ldo % 8 == 0 but N % 8 != 0, so a row mixes
                       full and partial 8-column groups
  wgmma_direct_scalar  kernel 2, per-element epilogue: out offset by one element or an odd ldo
  wgmma_fp32           kernel 2, fp32 out (never staged, never tailed)
  wgmma_tail           kernel 2, the partly filled last wave cut along K and summed in fp32 through the workspace
  wgmma_splitk         kernel 2, uniform split-K accumulated with bf16 red.global.add (weight gradients)

Recipes:
  plain    out = A.B^T
  full     bias + act + aux_out (pre-activation) + a separate residual, alpha = 0.5
  dgrad    out = (A.B^T) * act'(aux_in)
  dropout  bias + act + dropout 0.1 (seed from a device counter) + residual
  accum    out += A.B^T (residual is out)
"""
from __future__ import annotations

import dataclasses
import itertools

PATHS = ("simt_thread", "simt_warp", "wgmma_staged", "wgmma_direct_vec", "wgmma_direct_scalar", "wgmma_fp32", "wgmma_tail",
         "wgmma_splitk")
RECIPES = ("plain", "full", "dgrad", "dropout", "accum")
STAGED_PATHS = ("wgmma_staged", "wgmma_tail", "wgmma_splitk")
SM_BUDGETS = (132, 114)          # H100 SXM5, H100 PCIe
DROPOUT_P = 0.1
MAJORS = tuple(itertools.product((False, True), (False, True)))


def _up8(n):
    return (n + 7) // 8 * 8


@dataclasses.dataclass(frozen=True)
class Case:
    path: str
    M: int
    N: int
    K: int
    a_mn: bool
    b_mn: bool
    recipe: str
    act: int
    out_fp32: bool
    alpha: float
    # row strides (elements) and element offsets of each matrix inside its buffer
    lda: int
    ldb: int
    ldo: int
    ldr: int
    ld_aux: int
    a_off: int
    b_off: int
    out_off: int
    res_off: int
    aux_off: int
    pcie_path: str = ""          # the path on 114 SMs, where it differs (a few legacy weight-gradient shapes)

    def path_at(self, sms):
        return self.pcie_path if (self.pcie_path and sms < 132) else self.path

    @property
    def id(self):
        s = (f"{self.path}-{self.M}x{self.N}x{self.K}-{'a' if self.a_mn else 'A'}{'b' if self.b_mn else 'B'}-{self.recipe}"
             f"-act{self.act}")
        if self.a_off or self.b_off:
            s += f"-off{self.a_off}.{self.b_off}"
        if self.out_off % 8:
            s += f"-ooff{self.out_off}"
        if self.ldo % 2:
            s += f"-ldo{self.ldo}"
        if self.lda % 2 or self.ldb % 2:
            s += f"-ld{self.lda}.{self.ldb}"
        if self.alpha != 1.0:
            s += f"-alpha{self.alpha:g}"
        return s

    @property
    def residual_is_out(self):
        return self.recipe == "accum"

    @property
    def has_bias(self):
        return self.recipe in ("full", "dropout")

    @property
    def has_residual(self):
        return self.recipe in ("full", "dropout", "accum")


def make(path, M, N, K, a_mn=False, b_mn=False, recipe="plain", act=0, *, alpha=None, odd_lda=False, a_off=0,
         out_off=8, odd_ldo=False, pcie_path=""):
    """A case with distinct, aligned strides: lda = R8+8, ldb = R8+16 (R8 = the operand's row length rounded up to 8), ldo = N8+8, ldr = N8+24, ld_aux = N8+40
    (N8 = N rounded up to 8), so ldr > ldo and ld_aux > ldo and the staged epilogue still runs; outputs start 8 elements
    into their buffers.  odd_lda / a_off / out_off / odd_ldo break alignment to reach the SIMT and scalar paths."""
    n8 = _up8(N)
    lda = _up8(M if a_mn else K) + 8 + (1 if odd_lda else 0)
    ldb = _up8(N if b_mn else K) + 16
    ldo = n8 + 8 + (1 if odd_ldo else 0)
    if alpha is None:
        alpha = 0.5 if recipe == "full" else 1.0
    if recipe in ("plain", "accum"):
        act = 0
    return Case(path, M, N, K, a_mn, b_mn, recipe, act, path == "wgmma_fp32", alpha, lda, ldb, ldo,
                ldo if recipe == "accum" else n8 + 24, n8 + 40, a_off, 0, out_off,
                out_off if recipe == "accum" else 8, 8, pcie_path)


def staging(c):
    """(vec_ok, staged_ok) of dvla_gemm for this case, restated from csrc/gemm_sm90.cu:795-801: vec_ok needs every output-side
    pointer 16-byte aligned and its row stride a multiple of 8 elements (of 4 for an fp32 out / residual); staged_ok is
    vec_ok with a bf16 out and N % 8 == 0.  Buffers are 16-byte aligned, so an element offset aligns iff it does."""
    oal = 4 if c.out_fp32 else 8
    esz = 4 if c.out_fp32 else 2
    vec = (c.out_off * esz) % 16 == 0 and c.ldo % oal == 0
    if c.has_residual:
        vec = vec and (c.res_off * esz) % 16 == 0 and c.ldr % oal == 0
    if c.recipe in ("full", "dgrad"):                     # aux_out / aux_in
        vec = vec and (c.aux_off * 2) % 16 == 0 and c.ld_aux % 8 == 0
    return vec, vec and not c.out_fp32 and c.N % 8 == 0


def path_of(info, c):
    """The path a plan (dvla_gemm_plan_info) takes for case c."""
    if info.kernel == 0:
        return "simt_thread"
    if info.kernel == 1:
        return "simt_warp"
    assert info.kernel == 2, info.kernel
    if info.k_splits > 1:
        return "wgmma_splitk" if info.atomic_out else "wgmma_splitk_without_atomics"
    if info.tail_splits > 1:
        return "wgmma_tail"
    if c.out_fp32:
        return "wgmma_fp32"
    vec, staged = staging(c)
    if staged:
        return "wgmma_staged"
    return "wgmma_direct_vec" if vec else "wgmma_direct_scalar"


# Shapes per path.  Edges: M = 1 and M tails of 1, 64 and 127 rows past a multiple of 128; N % 128 tails and N % 8 != 0
# where the path allows it; K = 8 and K % 64 of 8 and 56; K > 2048 for split-K.
SHAPES = {
    "simt_thread": [(20, 1024, 6), (37, 13, 5), (1024, 6, 20), (13, 5, 37), (1, 136, 72), (255, 520, 120), (129, 1001, 8),
                    (192, 264, 56)],
    "simt_warp": [(7, 768, 960), (960, 7, 768), (129, 136, 184), (1, 1001, 1080), (255, 264, 128), (192, 13, 312)],
    "wgmma_staged": [(128, 128, 64), (256, 512, 256), (200, 264, 72), (300, 520, 256), (1, 136, 8), (129, 392, 120),
                     (192, 256, 1080), (255, 136, 184)],
    "wgmma_direct_vec": [(300, 1001, 256), (255, 135, 72), (1, 13, 8), (192, 263, 120), (129, 1001, 184), (64, 300, 1080)],
    "wgmma_direct_scalar": [(960, 7, 768), (129, 264, 72), (1, 520, 8), (255, 136, 120), (192, 1001, 184), (64, 7, 1080)],
    "wgmma_fp32": [(300, 520, 256), (129, 136, 72), (1, 264, 8), (255, 1001, 120), (192, 7, 184), (64, 384, 1080)],
    # a whole first wave plus a partial one, enough k-blocks for the fp32 fix-up to pay (at 132 and 114 SMs)
    "wgmma_tail": [(2580, 1024, 4096), (2433, 1000, 4104), (2368, 1096, 4168), (2431, 1000, 3640)],
    "wgmma_splitk": [(1024, 1024, 10320), (520, 264, 4104), (128, 136, 2056), (1153, 776, 6200)],
}


def _cross():
    cases = []
    for path in PATHS:
        shapes = SHAPES[path]
        recipes = ("accum",) if path == "wgmma_splitk" else \
            ("plain", "full", "dgrad", "dropout") if path == "wgmma_tail" else RECIPES   # a tail accumulation splits K
        i = 0
        for (a_mn, b_mn) in MAJORS:
            for recipe in recipes:
                M, N, K = shapes[i % len(shapes)]
                kw = {}
                if path == "simt_thread":
                    kw = {"a_off": 1} if i % 2 == 0 else {"odd_lda": True}
                elif path == "simt_warp":
                    kw = {"odd_lda": True}
                elif path == "wgmma_direct_scalar":
                    kw = {"out_off": 9} if i % 2 == 0 else {"odd_ldo": True}
                act = i % 6
                if recipe == "dgrad" and act == 0:       # act'(x) = 1 would leave aux_in unread
                    act = 4
                cases.append(make(path, M, N, K, a_mn, b_mn, recipe, act=act, **kw))
                i += 1
    return cases


def _legacy():
    """Every shape and epilogue the gemm_basic, gemm_epilogue, gemm_splitk and gemm_tail groups of tools/gpu_kernel_check.py
    check (there with contiguous operands and a whole-tensor L2 bar)."""
    cases = []
    for (M, N, K) in [(128, 128, 64), (256, 512, 256), (200, 264, 72)]:                     # gemm_basic
        for (a_mn, b_mn) in MAJORS:
            cases.append(make("wgmma_staged", M, N, K, a_mn, b_mn))
    for act in range(6):                                                                     # gemm_epilogue
        cases.append(make("wgmma_staged", 300, 520, 256, recipe="full", act=act, alpha=1.0))
        cases.append(make("wgmma_staged", 300, 520, 256, b_mn=True, recipe="dgrad", act=act))
    cases += [make("wgmma_fp32", 300, 520, 256, recipe="accum", alpha=0.5), make("wgmma_staged", 300, 520, 256, recipe="accum"),
              make("wgmma_staged", 300, 520, 256, recipe="dropout", act=0)]
    cases += [make("simt_thread", 20, 1024, 6, recipe="full", alpha=1.0, odd_lda=True),
              make("wgmma_direct_scalar", 960, 7, 768, recipe="full", alpha=1.0, odd_ldo=True),
              make("simt_thread", 37, 13, 5, recipe="full", alpha=1.0, odd_lda=True),
              make("simt_thread", 1024, 6, 20, True, True, odd_lda=True), make("simt_warp", 7, 768, 960, True, True, odd_lda=True),
              make("simt_thread", 13, 5, 37, True, True, odd_lda=True)]
    for (M, N, K) in [(1024, 1024, 10320), (1024, 1024, 42400), (1024, 3072, 10320), (3072, 1024, 10320),      # gemm_splitk
                      (1024, 768, 10320), (768, 768, 31520), (768, 3072, 31520), (2304, 768, 31520), (520, 264, 4104),
                      (128, 136, 2056)]:
        # the model's three largest split-K picks at 132 SMs find one split no slower at 114 and run whole tiles there
        pcie = "wgmma_staged" if (M, N, K) in ((1024, 3072, 10320), (3072, 1024, 10320), (2304, 768, 31520)) else ""
        cases.append(make("wgmma_splitk", M, N, K, True, True, "accum", pcie_path=pcie))
    # gemm_tail: only 2580 x 1024 x 4096 forms a split tail; the others are whole waves or too short in K for one to pay
    for (M, N, K, b_mn, path) in [(10320, 1024, 4096, False, "wgmma_staged"), (10320, 1024, 4096, True, "wgmma_staged"),
                                  (10320, 1024, 3072, False, "wgmma_staged"), (10320, 1024, 1024, True, "wgmma_staged"),
                                  (2580, 1024, 4096, False, "wgmma_tail"), (1300, 512, 2048, False, "wgmma_staged"),
                                  (5000, 1000, 1536, True, "wgmma_staged"), (31520, 768, 3072, False, "wgmma_staged")]:
        cases.append(make(path, M, N, K, False, b_mn, "plain"))
        cases.append(make(path, M, N, K, False, b_mn, "full", act=2, alpha=1.0))
    cases.append(make("wgmma_staged", 10320, 1024, 4096, recipe="dropout", act=0))
    return cases


def _unique(cases):
    seen, out = set(), []
    for c in cases:
        if c not in seen:
            seen.add(c)
            out.append(c)
    ids = [c.id for c in out]
    assert len(set(ids)) == len(ids), "case ids must be unique"
    return out


CASES = _unique(_cross() + _legacy())
