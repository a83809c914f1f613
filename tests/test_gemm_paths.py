"""Dense projections (`gemm.linear`, `gemm.linear_train`) on every route and every kernel instance, against float64.

`predict_route` restates the rule of gemm.py; the routes:
  L0 F.linear in fp32            "auto" with rows <= SMALL_M; MODE "fp32"; K % 4 != 0; inputs that are not fp32 CUDA
                                 tensors on the current device, and empty inputs
  L1 gemm_f16x3_pre              "auto", OWN_KERNEL "f16x3", K % 64 == 0
  L2 gemm_3xtf32_pre             "tcgen05"; "auto" with K % 32 == 0 and K % 64 != 0, or OWN_KERNEL "tf32x3"
  L3 gemm_3xtf32 ("SS")          LONG_K_PRESPLIT and K >= 1024
  L4 gemm_3xtf32_raw             PRESPLIT_PERSISTENT False
  L5 split_tf32 + one cuBLAS TF32 GEMM over 3K     MODE "3xtf32", or an own-kernel mode with K % 32 != 0
  L6 L5 with one GEMM per K chunk of K_CHUNK       K > K_CHUNK and K % K_CHUNK == 0
  L7 single-pass TF32 F.linear   MODE "tf32"
  T1 _LinearF16x3, dx on the 3xFP16 kernel over the W^T split      linear_train, N % 64 == 0
  T2 _LinearF16x3, dx on cuBLAS                                    linear_train, N % 64 != 0
  T3 F.linear                                                      every other linear_train call
The GPU route test wraps the `cabi` entry points and F.linear in call-through recorders and checks that exactly the
predicted one ran.

L1-L4 end in one kernel template, gemm3x_kernel<F16, SPLIT_W> (csrc/wgmma.cuh), in four instances: fp16 pieces with a
fixed activation scale (gemm_f16x3_pre) or device scales (gemm_f16x3_scaled, the training path), TF32 pieces with a
pre-split weight (gemm_3xtf32_pre and gemm_3xtf32) or one split in the kernel (gemm_3xtf32_raw).  Each is run through its
C entry point at M, N and K tails around the 128 x 128 tile and the ring depth, with the fused input activations, a
row pitch above K, the scalar epilogue (odd ldc, C not 8-byte aligned) and capped persistent grids, on inputs with mixed
magnitudes, exact zeros, constant rows, one large element among small ones and weights over six decades.

Bounds are element-wise: |got - ref| <= c * 2^-24 * S + floor, ref = F.linear in float64 on act(x) and S the same on
|act(x)| and |W| (plus |b|): the error of a float32 sum of products is a multiple of 2^-24 times the sum of the absolute
products whatever the sign pattern.  The floor is the absolute resolution of the fp16 pieces, 2^-25 per operand element
divided by its power-of-two scale (2^-29 |W| for the fixed activation scale 16: include/sdetr_b200.h).

Non-finite inputs: a NaN (four encodings: GPU arithmetic makes 0x7fffffff, which a carry through the exponent of a naive
TF32 rounding turns into -0) or an inf at one element of x or W must make exactly the outputs float64 F.linear makes
non-finite non-finite, and leave every other output bit-identical to the clean run."""
import math
import os

import pytest
import torch

F = torch.nn.functional
DEV = "cuda:0"
U = 2.0 ** -24  # unit round-off of float32

# Bound constants c of |got - ref| <= c * 2^-24 * S + floor.  Each is about four times the largest c observed over every
# case of this file on an H100 80GB HBM3 at 700 W (noted beside it).
C_F16 = 52.0    # gemm_f16x3_pre / _scaled: the instances, route L1, linear_train's y and dx (observed 13.0, gemm_f16x3_pre;
                #   dx at dy scales 1, 1e-12: 4.4, 4.0; at 1e-20 the fp16 floor of dy's clamped scale covers all of it)
C_TF32 = 60.0   # gemm_3xtf32_pre / gemm_3xtf32 / gemm_3xtf32_raw and route L2 (observed 15.3)
C_SPLIT = 100.0  # split_tf32 + cuBLAS TF32 over 3K, route L5 (observed 25.4)
C_FP32 = 25.0   # cuBLAS SGEMM: route L0, and dx (T2), dW, db of linear_train (observed 6.0, 5.1, 0.71, 0.19)
C_TF32_1 = 4.0  # single-pass TF32 (MODE "tf32"), in units of 2^-11 (observed 1.04)

OBSERVED = {}


def _observe(name, err, scale, floor=0.0):
    """Record the c an error needs (err - floor) / (2^-24 S); printed at the end with SDETR_GEMM_OBSERVE=1 (calibration)."""
    need = ((err - floor).clamp_min(0) / scale.clamp_min(1e-300)).masked_fill(scale == 0, 0)
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), float(need.max()) if need.numel() else 0.0)


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    if os.environ.get("SDETR_GEMM_OBSERVE"):
        print("\nOBSERVED", {k: round(v, 3) for k, v in sorted(OBSERVED.items())})


@pytest.fixture(scope="module")
def gemm():
    import salience_detr_b200 as p
    return p.gemm


@pytest.fixture(autouse=True)
def _restore(gemm):
    """Every test starts from and leaves the shipped routing switches, an uncapped persistent grid and torch's TF32
    setting."""
    saved = (gemm.MODE, gemm.OWN_KERNEL, gemm.LONG_K_PRESPLIT, gemm.PRESPLIT_PERSISTENT, torch.backends.cuda.matmul.allow_tf32)
    yield
    gemm.MODE, gemm.OWN_KERNEL, gemm.LONG_K_PRESPLIT, gemm.PRESPLIT_PERSISTENT = saved[:4]
    torch.backends.cuda.matmul.allow_tf32 = saved[4]
    if torch.cuda.is_available():
        gemm.cabi.lib().sdetr_set_persistent_ctas(0)


# ---- the routing rule -----------------------------------------------------------------------------------------------
SMALL_M, K_CHUNK = 2304, 512


def predict_route(mode, own, long_k, persistent, rows, K, N=64, native=True, train=False):
    """Which route gemm.linear (train=False) or gemm.linear_train (train=True) takes.  `native`: x, W and b are fp32
    CUDA tensors on the current device (any layout)."""
    if train:
        if mode == "auto" and own == "f16x3" and native and rows > SMALL_M and K % 64 == 0:
            return "T1" if N % 64 == 0 else "T2"
        return "T3"
    if (mode == "auto" and rows <= SMALL_M) or not native or rows == 0:
        return "L0"
    if mode in ("tcgen05", "auto") and K % 32 == 0:
        if K >= 1024 and long_k:
            return "L3"
        if own == "f16x3" and mode == "auto" and K % 64 == 0:
            return "L1"
        return "L2" if persistent else "L4"
    if mode == "fp32" or K % 4 != 0:
        return "L0"
    if mode == "tf32":
        return "L7"
    return "L6" if K > K_CHUNK and K % K_CHUNK == 0 else "L5"


ROUTES = ("L0", "L1", "L2", "L3", "L4", "L5", "L6", "L7", "T1", "T2", "T3")
# (mode, OWN_KERNEL, LONG_K_PRESPLIT, PRESPLIT_PERSISTENT, rows, K, N, input kind, train)
ROUTE_CASES = [
    ("auto", "f16x3", False, True, SMALL_M, 64, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 32, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 96, 91, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 100, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 576, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 1024, 64, "f32", False),
    ("auto", "f16x3", True, True, SMALL_M + 1, 1024, 64, "f32", False),
    ("auto", "f16x3", True, True, SMALL_M + 1, 576, 64, "f32", False),
    ("auto", "tf32x3", False, True, SMALL_M + 1, 64, 64, "f32", False),
    ("auto", "tf32x3", False, False, SMALL_M + 1, 2048, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 30, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 64, "f64", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 64, "transposed", False),
    ("tcgen05", "f16x3", False, True, 10, 64, 64, "f32", False),
    ("tcgen05", "f16x3", False, False, 10, 2048, 64, "f32", False),
    ("tcgen05", "f16x3", True, True, 10, 2048, 64, "f32", False),
    ("tcgen05", "f16x3", False, True, 10, 100, 64, "f32", False),
    ("tcgen05", "f16x3", False, True, 0, 64, 64, "f32", False),
    ("tcgen05", "f16x3", False, True, 10, 64, 64, "cpu", False),
    ("tcgen05", "f16x3", False, True, 10, 64, 64, "odd_pitch", False),
    ("3xtf32", "f16x3", False, True, 10, 512, 64, "f32", False),
    ("3xtf32", "f16x3", False, True, 10, 576, 64, "f32", False),
    ("3xtf32", "f16x3", False, True, 10, 1024, 64, "f32", False),
    ("3xtf32", "f16x3", False, True, 10, 2048, 64, "misaligned", False),
    ("3xtf32", "f16x3", False, True, 10, 100, 64, "transposed", False),
    ("fp32", "f16x3", False, True, SMALL_M + 1, 64, 64, "f32", False),
    ("tf32", "f16x3", False, True, SMALL_M + 1, 64, 64, "f32", False),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 128, "f32", True),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 128, "misaligned", True),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 91, "transposed", True),
    ("auto", "f16x3", False, True, SMALL_M, 64, 128, "f32", True),
    ("auto", "f16x3", False, True, SMALL_M + 1, 96, 128, "f32", True),
    ("auto", "tf32x3", False, True, SMALL_M + 1, 64, 128, "f32", True),
    ("tcgen05", "f16x3", False, True, SMALL_M + 1, 64, 128, "f32", True),
    ("auto", "f16x3", False, True, SMALL_M + 1, 64, 128, "f64", True),
]


def _route_of(case):
    mode, own, long_k, persistent, rows, K, N, kind, train = case
    return predict_route(mode, own, long_k, persistent, rows, K, N, native=kind not in ("f64", "cpu"), train=train)


def test_route_table_reaches_every_route(gemm):
    """The case table reaches every route, predict_route's thresholds are gemm.py's, and the boundary rows / K values are
    in it."""
    assert (gemm.SMALL_M, gemm.K_CHUNK) == (SMALL_M, K_CHUNK)
    assert {_route_of(c) for c in ROUTE_CASES} == set(ROUTES)
    assert {c[4] for c in ROUTE_CASES} >= {SMALL_M, SMALL_M + 1}
    assert {c[5] for c in ROUTE_CASES} >= {32, 64, 96, 100, 576, 1024, 2048}


def test_predict_route_rule():
    """Spot checks of the restated rule at its edges."""
    assert predict_route("auto", "f16x3", False, True, SMALL_M, 64) == "L0"
    assert predict_route("auto", "f16x3", False, True, SMALL_M + 1, 64) == "L1"
    assert predict_route("auto", "f16x3", False, True, SMALL_M + 1, 96) == "L2"
    assert predict_route("auto", "f16x3", True, True, SMALL_M + 1, 1024) == "L3"
    assert predict_route("auto", "f16x3", True, True, SMALL_M + 1, 960) == "L1"
    assert predict_route("tcgen05", "f16x3", False, True, 1, 64) == "L2"
    assert predict_route("tcgen05", "f16x3", False, False, 1, 64) == "L4"
    assert predict_route("tcgen05", "f16x3", False, True, 1, 36) == "L5"
    assert predict_route("tcgen05", "f16x3", False, True, 1, 34) == "L0"
    assert predict_route("3xtf32", "f16x3", True, True, 1, 1024) == "L6"
    assert predict_route("3xtf32", "f16x3", False, True, 1, 1536) == "L6"
    assert predict_route("3xtf32", "f16x3", False, True, 1, 1000) == "L5"
    assert predict_route("tf32", "f16x3", False, True, 1, 64) == "L7"
    assert predict_route("fp32", "f16x3", False, True, 10 ** 6, 64) == "L0"
    assert predict_route("3xtf32", "f16x3", False, True, 10 ** 6, 64, native=False) == "L0"
    assert predict_route("tcgen05", "f16x3", False, True, 0, 64) == "L0"
    assert predict_route("auto", "f16x3", False, True, SMALL_M + 1, 64, 192, train=True) == "T1"
    assert predict_route("auto", "f16x3", False, True, SMALL_M + 1, 64, 100, train=True) == "T2"
    assert predict_route("auto", "f16x3", False, True, SMALL_M + 1, 32, 128, train=True) == "T3"


@pytest.mark.parametrize("mode", ["auto", "tcgen05", "3xtf32", "fp32", "tf32"])
def test_cpu_and_other_dtypes_are_f_linear(gemm, mode):
    """CPU tensors and non-fp32 inputs go to F.linear in every mode (no CUDA needed): the same result bit for bit."""
    gemm.MODE = mode
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float32, torch.float64, torch.bfloat16):
        for rows in (0, 1, SMALL_M + 1):
            x = torch.randn(rows, 64, generator=g).to(dtype)
            w = torch.randn(96, 64, generator=g).to(dtype)
            b = torch.randn(96, 2, generator=g).to(dtype)[:, 0]  # a non-contiguous bias
            assert torch.equal(gemm.linear(x, w, b), F.linear(x, w, b))
            assert torch.equal(gemm.linear(x, w, b, relu_input=True), F.linear(F.relu(x), w, b))
            assert torch.equal(gemm.linear_train(x, w, b), F.linear(x, w, b))


# ---- inputs ---------------------------------------------------------------------------------------------------------
NONFINITE = {"nan_7fc00000": 0x7FC00000, "nan_7fffffff": 0x7FFFFFFF, "nan_ffc00000": 0xFFC00000 - 2 ** 32,
             "nan_ffffffff": -1, "+inf": math.inf, "-inf": -math.inf}


def _poke(t, idx, v):
    """t[idx] = v with the exact bit pattern (an int is a float32 encoding)."""
    if isinstance(v, int):
        t.view(torch.int32)[idx] = v
    else:
        t[idx] = v


def make_x(kind, M, K, g):
    if kind == "mixed":  # magnitudes 2^-7 .. 4000 inside every row, random signs
        mag = torch.exp2(torch.rand(M, K, generator=g) * (math.log2(4000) + 7) - 7)
        return mag * torch.randint(0, 2, (M, K), generator=g).mul(2).sub(1)
    x = torch.randn(M, K, generator=g)
    if kind == "zeros":  # exact zero rows and columns
        x[::3] = 0
        x[:, ::5] = 0
    elif kind == "const":  # constant rows
        x = x[:, :1].expand(M, K).contiguous()
    elif kind == "spike":  # one large element among small ones in every row
        x = x * 1e-3
        x[torch.arange(M), torch.randint(0, K, (M,), generator=g)] = 3000.0
    return x


def make_w(kind, N, K, g):
    w = torch.randn(N, K, generator=g) / K ** 0.5
    if kind == "wide":  # six decades of dynamic range
        w = w * torch.logspace(-6, 0, K)[torch.randperm(K, generator=g)]
    return w


def _act64(x, act):
    x = x.double()
    return F.relu(x) if act == 1 else F.gelu(x) if act == 2 else x


def ref_and_scale(x, w, b, act):
    """float64 F.linear on act(x) and the bound's S (the same on absolute values)."""
    xa, w64 = _act64(x, act), w.double()
    b64 = None if b is None else b.double()
    return F.linear(xa, w64, b64), F.linear(xa.abs(), w64.abs(), None if b64 is None else b64.abs())


def check_bound(name, got, x, w, b, act, c, a_scale=None, w_scale=None):
    """|got - ref| <= c 2^-24 S + floor, element-wise; a_scale / w_scale: the fp16 pieces' power-of-two scales."""
    ref, S = ref_and_scale(x, w, b, act)
    floor = torch.zeros_like(ref)
    if a_scale is not None:
        xa, w64 = _act64(x, act).abs(), w.double().abs()
        floor = 2.0 ** -25 * (w64.sum(1)[None, :] / a_scale + xa.sum(1)[:, None] / w_scale)
    err = (got.double() - ref).abs()
    _observe(name, err, U * S, floor)
    bad = ~(err <= c * U * S + floor)
    assert not bad.any(), (name, int(bad.sum()), float(((err - floor) / (U * S)).max()))


# ---- the kernel instances through their C entry points ----------------------------------------------------------------
INSTANCES = ("f16_pre", "f16_scaled", "tf32_pre", "tf32_ss", "tf32_raw")
C_OF = {"f16_pre": C_F16, "f16_scaled": C_F16, "tf32_pre": C_TF32, "tf32_ss": C_TF32, "tf32_raw": C_TF32}


def run_instance(cabi, inst, x, w, b, act, C=None):
    """C = act(x) W^T + b through the instance's C entry point -> (C, a_scale, w_scale); x (M, K) with unit last stride,
    C an (M, N) tensor with unit column stride (fresh when None)."""
    lib, stream = cabi.lib(), cabi._stream()
    M, K = x.shape
    N = w.shape[0]
    if C is None:
        C = torch.empty(M, N, device=DEV)
    lda, ldc = (x.stride(0) if M > 1 else K), (C.stride(0) if M > 1 else N)
    bp = None if b is None else b.data_ptr()
    a_scale = w_scale = None
    if inst == "f16_pre":
        hi, lo, w_scale = cabi.split_f16_pair(w)
        a_scale = 16.0
        rc = lib.sdetr_gemm_f16x3_pre(x.data_ptr(), lda, hi.data_ptr(), lo.data_ptr(), float(w_scale), bp, C.data_ptr(), ldc,
                                      M, N, K, act, stream)
    elif inst == "f16_scaled":
        assert act == 0
        a = cabi.pow2_scale(x.contiguous(), 12)
        hi, lo, ws = cabi.split_f16_pair_dev(w)
        rc = lib.sdetr_gemm_f16x3_scaled(x.data_ptr(), lda, a.data_ptr(), hi.data_ptr(), lo.data_ptr(), ws.data_ptr(), bp,
                                         C.data_ptr(), ldc, M, N, K, stream)
        a_scale, w_scale = a.item(), ws.item()
    elif inst == "tf32_raw":
        wc = w.contiguous()
        rc = lib.sdetr_gemm_3xtf32_raw(x.data_ptr(), lda, wc.data_ptr(), bp, C.data_ptr(), ldc, M, N, K, act, stream)
    else:
        hi, lo = cabi.split_tf32_pair(w)
        fn = lib.sdetr_gemm_3xtf32_pre if inst == "tf32_pre" else lib.sdetr_gemm_3xtf32
        rc = fn(x.data_ptr(), lda, hi.data_ptr(), lo.data_ptr(), bp, C.data_ptr(), ldc, M, N, K, act, stream)
    cabi._check(rc, inst)
    return C, a_scale, w_scale


M_TAILS = (1, 2, 63, 64, 65, 127, 128, 129)
N_TAILS = (1, 2, 3, 91, 127, 128, 129, 300)
K_BLOCKS = {True: (64, 128, 192, 256, 2048), False: (32, 96, 128, 160, 2048)}  # 3-stage f16 / 4-stage tf32 rings
X_KINDS = ("randn", "mixed", "zeros", "const", "spike")


def kernel_cases(inst):
    """(M, N, K, act, bias, pitched x, x kind, w kind): the M tails, the N tails, the k-block counts and one size with
    several tiles per CTA, with the activation, bias, row pitch and input kinds rotating through them."""
    ks = K_BLOCKS[inst.startswith("f16")]
    shapes = ([(M, 129, ks[i % 5]) for i, M in enumerate(M_TAILS)] + [(130, N, ks[i % 5]) for i, N in enumerate(N_TAILS)] +
              [(65, 128, K) for K in ks] + [(40000, 300, ks[1])])
    return [(M, N, K, 0 if inst == "f16_scaled" else i % 3, i % 2 == 0, i % 4 == 1, X_KINDS[i % 5], ("randn", "wide")[i // 5 % 2])
            for i, (M, N, K) in enumerate(shapes)]


@pytest.fixture(scope="module")
def cabi():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p.cabi


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTANCES)
def test_kernel_instance_bounds(cabi, inst):
    """Every instance within its element-wise bound of float64 at the tail / k-block / activation / bias / pitch cases."""
    g = torch.Generator().manual_seed(11)
    for M, N, K, act, bias, pitched, xk, wk in kernel_cases(inst):
        x = make_x(xk, M, K, g)
        w, b = make_w(wk, N, K, g), (torch.randn(N, generator=g) if bias else None)
        x, w, b = x.to(DEV), w.to(DEV), None if b is None else b.to(DEV)
        if pitched:  # rows of a wider buffer
            wide = torch.randn(M, K + 32, device=DEV)
            wide[:, :K] = x
            x = wide[:, :K]
        got, a_s, w_s = run_instance(cabi, inst, x, w, b, act)
        check_bound(inst, got, x, w, b, act, C_OF[inst], a_s, w_s)


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTANCES)
def test_kernel_instance_epilogue_and_grid(cabi, inst):
    """The scalar epilogue (odd ldc; C 4 bytes past an 8-byte boundary) writes the same bits as the paired one and nothing
    outside C; persistent grids capped at 1, 2, 7, tiles - 1 and tiles + 1 CTAs and repeated calls give the same bits."""
    g = torch.Generator().manual_seed(12)
    K = 128 if inst.startswith("f16") else 96
    act = 0 if inst == "f16_scaled" else 2
    M, N = 1000, 300  # 8 x 3 = 24 tiles
    x, w, b = (torch.randn(M, K, generator=g).to(DEV), make_w("randn", N, K, g).to(DEV), torch.randn(N, generator=g).to(DEV))
    want = run_instance(cabi, inst, x, w, b, act)[0]
    for width, col in ((N + 3, 1), (N + 5, 1), (N + 4, 1), (N + 3, 2)):  # ldc odd / base +4 bytes, ldc even / base +4
        big = torch.full((M, width), 7.0, device=DEV)
        C = big[:, col:col + N]
        run_instance(cabi, inst, x, w, b, act, C)
        assert torch.equal(C, want), (inst, width, col)
        outside = torch.ones_like(big, dtype=torch.bool)
        outside[:, col:col + N] = False
        assert (big[outside] == 7.0).all(), (inst, width, col)
    tiles = 8 * 3
    try:
        for cap in (1, 2, 7, tiles - 1, tiles + 1, 0):
            cabi.lib().sdetr_set_persistent_ctas(cap)
            for _ in range(2):
                assert torch.equal(run_instance(cabi, inst, x, w, b, act)[0], want), (inst, cap)
    finally:
        cabi.lib().sdetr_set_persistent_ctas(0)


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTANCES)
def test_kernel_instance_nonfinite(cabi, inst):
    """A NaN (four encodings) or an inf at one element of x -- and of W for the instances that split W on the device --
    makes exactly the outputs float64 F.linear makes non-finite non-finite, with every activation, and leaves every
    other output bit-identical to the clean run."""
    g = torch.Generator().manual_seed(13)
    K = 128 if inst.startswith("f16") else 96
    M, N, r, n, k = 200, 130, 131, 129, 67
    x0, w0, b = (torch.randn(M, K, generator=g).to(DEV), make_w("randn", N, K, g).to(DEV), torch.randn(N, generator=g).to(DEV))
    x0[r, k], w0[n, k] = 0.5, 0.01  # not the maximum: the device scales of f16_scaled come from the other entries
    for act in ((0,) if inst == "f16_scaled" else (0, 1, 2)):
        clean = run_instance(cabi, inst, x0, w0, b, act)[0]
        targets = ("x",) if inst == "f16_pre" else ("x", "w")  # split_f16_pair refuses a non-finite weight on the host
        for name, v in NONFINITE.items():
            for target in targets:
                x, w = x0.clone(), w0.clone()
                _poke(x if target == "x" else w, (r, k) if target == "x" else (n, k), v)
                got = run_instance(cabi, inst, x, w, b, act)[0]
                ref = F.linear(_act64(x, act), w.double(), b.double())
                assert torch.equal(got.isfinite(), ref.isfinite()), (inst, act, name, target)
                keep = torch.ones_like(got, dtype=torch.bool)
                if target == "x":
                    keep[r] = False
                else:
                    keep[:, n] = False
                assert torch.equal(got[keep], clean[keep]), (inst, act, name, target)


@pytest.mark.gpu
def test_f16_fixed_scale_range(cabi):
    """gemm_f16x3_pre and the fused FFN take |x| < 4094 at full accuracy; from 4096 on a row comes out non-finite,
    never finite and wrong."""
    g = torch.Generator().manual_seed(14)
    K, N, M = 256, 256, 70
    w = make_w("randn", N, K, g).to(DEV)
    w1, b1 = make_w("randn", 512, 256, g).to(DEV), torch.randn(512, generator=g).to(DEV)
    w2, b2 = make_w("randn", 256, 512, g).to(DEV), torch.randn(256, generator=g).to(DEV)
    s1, s2 = cabi.split_f16_pair(w1), cabi.split_f16_pair(w2)
    for v, ok in ((4093.9, True), (-4093.9, True), (4096.0, False), (-5000.0, False), (1e6, False), (3.0e38, False)):
        x = torch.randn(M, K, generator=g).to(DEV)
        x[5, 17] = v
        got, a_s, w_s = run_instance(cabi, "f16_pre", x, w, None, 0)
        if ok:
            check_bound("f16_pre", got, x, w, None, 0, C_F16, a_s, w_s)
        else:
            assert not got[5].isfinite().any(), v
            assert got[torch.arange(M) != 5].isfinite().all()
        y = cabi.ffn_fused_layernorm(x, s1, b1, s2, b2)
        if ok:
            h = F.relu(F.linear(x.double(), w1.double(), b1.double()))
            err = (y.double() - F.linear(h, w2.double(), b2.double())).abs()
            assert (err <= 1e-4 * (1 + F.linear(h, w2.double().abs()).abs())).all()
        else:
            assert not y[5].isfinite().any(), v
            assert y[torch.arange(M) != 5].isfinite().all()


@pytest.mark.gpu
def test_ffn_fused_nonfinite(cabi):
    """The fused FFN, bare and with its LayerNorm: a NaN or inf in a row of x makes that row non-finite (the hidden ReLU
    propagates NaN like torch.relu) and leaves every other row bit-identical."""
    g = torch.Generator().manual_seed(15)
    M, r, k = 200, 77, 3
    w1, b1 = make_w("randn", 1024, 256, g).to(DEV), torch.randn(1024, generator=g).to(DEV)
    w2, b2 = make_w("randn", 256, 1024, g).to(DEV), torch.randn(256, generator=g).to(DEV)
    gamma, beta = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV), (0.1 * torch.randn(256, generator=g)).to(DEV)
    s1, s2 = cabi.split_f16_pair(w1), cabi.split_f16_pair(w2)
    x0 = torch.randn(M, 256, generator=g).to(DEV)
    for ln in (False, True):
        extra = (gamma, beta, 1e-5) if ln else ()
        clean = cabi.ffn_fused_layernorm(x0, s1, b1, s2, b2, *extra)
        for name, v in NONFINITE.items():
            x = x0.clone()
            _poke(x, (r, k), v)
            y = cabi.ffn_fused_layernorm(x, s1, b1, s2, b2, *extra)
            h = F.linear(F.relu(F.linear(x.double(), w1.double(), b1.double())), w2.double(), b2.double())
            ref = F.layer_norm(x.double() + h, (256,), gamma.double(), beta.double(), 1e-5) if ln else h
            assert torch.equal(y.isfinite(), ref.isfinite()), (ln, name)
            rows = torch.arange(M, device=DEV) != r
            assert torch.equal(y[rows], clean[rows]), (ln, name)


# ---- the split kernels ------------------------------------------------------------------------------------------------
def tf32_rna_bits(x):
    """Round-to-nearest, ties away from zero, on the low 13 bits of float32 x (as int64 bit patterns); NaN and inf
    unchanged."""
    u = x.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (u + 0x1000) & 0xFFFFE000
    return torch.where((u & 0x7F800000) == 0x7F800000, u, r)


def _as_f32(bits):
    return torch.where(bits >= 2 ** 31, bits - 2 ** 32, bits).to(torch.int32).view(torch.float32)


def special_values(g):
    b = [0, 0x80000000, 1, 0x80000001, 0x7FFFFF, 0x807FFFFF, 0x7FF000, 0x801000, 0x00800000, 0x3F801000, 0xBF801000,
         0x3F803000, 0x3F800FFF, 0x3F801001, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7FF000, 0x7F7FEFFF, 0x7F7FE000, 0x7FC00000,
         0x7FFFFFFF, 0xFFC00000, 0xFFFFFFFF, 0x7F800001, 0x7F801000, 0x7F800000, 0xFF800000]
    rnd = torch.randint(0, 2 ** 32, (4096,), generator=g, dtype=torch.int64)
    return _as_f32(torch.cat([torch.tensor(b, dtype=torch.int64), rnd]))


@pytest.mark.gpu
def test_split_tf32_pair_bits(cabi):
    """split_tf32_pair: hi is the ties-away TF32 rounding of w bit for bit (NaN stays NaN, with its payload), lo the same
    rounding of w - hi; the in-kernel split of gemm_3xtf32_raw gives the pre-split results (test above) from the same
    arithmetic."""
    w = special_values(torch.Generator().manual_seed(16)).view(-1, 1)
    hi, lo = cabi.split_tf32_pair(w.to(DEV))
    hi, lo = hi.cpu(), lo.cpu()
    want_hi = _as_f32(tf32_rna_bits(w))
    assert torch.equal(hi.view(torch.int32), want_hi.view(torch.int32))
    d = w - want_hi  # float32 subtraction, as the kernel does it
    want_lo = _as_f32(tf32_rna_bits(d))
    fin = want_lo.isfinite()
    assert torch.equal(lo.isnan(), want_lo.isnan()) and torch.equal(lo.isinf(), want_lo.isinf())
    assert torch.equal(lo[fin].view(torch.int32), want_lo[fin].view(torch.int32))
    assert w.isnan().sum() > 0 and torch.equal(hi.isnan(), w.isnan())


@pytest.mark.gpu
def test_split_f16_pairs(cabi):
    """split_f16_pair and split_f16_pair_dev: hi = fp16_rn(s w), lo = fp16_rn(s w - hi), exactly."""
    g = torch.Generator().manual_seed(17)
    w = torch.randn(300, 67, generator=g) * torch.logspace(-6, 0, 67)
    w[0, :8] = torch.tensor([0.0, -0.0, 1.0, -1.0, 1 + 2 ** -11, 1 + 3 * 2 ** -11, 2 ** -20, 1e-30])  # fp16 ties, tiny values
    hi, lo, s = cabi.split_f16_pair(w.to(DEV))
    hd, ld, sd = cabi.split_f16_pair_dev(w.to(DEV))
    assert sd.item() == s
    for h, l in ((hi, lo), (hd, ld)):
        sw = w * s
        want_hi = sw.half()
        want_lo = (sw - want_hi.float()).half()
        assert torch.equal(h.cpu().view(torch.int16), want_hi.view(torch.int16))
        assert torch.equal(l.cpu().view(torch.int16), want_lo.view(torch.int16))


def pow2_ref(x, t):
    """2^s with max|finite x| * 2^s in [2^(t-1), 2^t), s clamped to [-60, 60]; 1 when there is no non-zero finite entry."""
    fin = x[x.isfinite()].double().abs()
    amax = float(fin.max()) if fin.numel() else 0.0
    if amax == 0:
        return 1.0
    return 2.0 ** max(-60, min(60, t - math.frexp(amax)[1]))


@pytest.mark.gpu
def test_pow2_scale(cabi):
    """pow2_scale on counts 1..5 and a multi-block count with a tail; all zeros, a subnormal maximum, an exact power of two,
    NaN and inf (the scale comes from the finite entries); back to back on one stream and on two streams."""
    g = torch.Generator().manual_seed(18)
    cases = [torch.randn(n, generator=g) for n in (1, 2, 3, 4, 5)]
    cases += [torch.randn(4 * 256 * 600 + 7, generator=g), torch.zeros(33), torch.full((9,), 1e-40),
              torch.tensor([0.25, -0.5, 0.125]), torch.tensor([-1024.0, 3.0]), torch.tensor([1e-20, -3e-21]),
              torch.tensor([1.0, float("nan"), 2.0, -3.0, 0.5]), torch.tensor([1.0, float("inf"), 2.0, -3.0, 0.5]),
              torch.tensor([float("-inf"), float("nan")]), torch.tensor([3.0e38, -1.0])]
    big = torch.randn(4 * 256 * 600 + 7, generator=g)
    big[123457] = float("inf")
    cases.append(big)
    for x in cases:
        for t in (12, 14):
            assert cabi.pow2_scale(x.to(DEV), t).item() == pow2_ref(x, t), (x[:5], t)
    a, b = torch.randn(1000, generator=g).to(DEV) * 1e5, torch.randn(3, generator=g).to(DEV) * 1e-5
    sa, sb = cabi.pow2_scale(a, 12), cabi.pow2_scale(b, 12)  # back to back: the second sees a reset state
    assert (sa.item(), sb.item()) == (pow2_ref(a.cpu(), 12), pow2_ref(b.cpu(), 12))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.current_stream().synchronize()
    with torch.cuda.stream(s1):
        ra = cabi.pow2_scale(a, 12)
    with torch.cuda.stream(s2):
        rb = cabi.pow2_scale(b, 12)
    torch.cuda.synchronize()
    assert (ra.item(), rb.item()) == (pow2_ref(a.cpu(), 12), pow2_ref(b.cpu(), 12))


# ---- routes through gemm.linear / gemm.linear_train ---------------------------------------------------------------------
ENTRY = ("gemm_f16x3_pre", "gemm_3xtf32_pre", "gemm_3xtf32", "gemm_3xtf32_raw", "split_tf32", "gemm_f16x3_scaled")


def _layout(kind, rows, K, g, dtype=torch.float32):
    """x (rows, K) in one of the layouts F.linear takes."""
    if kind == "transposed":
        return torch.randn(K, rows, generator=g).to(DEV).t()
    if kind == "odd_pitch":
        return torch.randn(rows, K + 1, generator=g).to(DEV)[:, :K]
    if kind == "misaligned":  # 4 bytes past a 16-byte boundary, pitch a multiple of 4
        return torch.randn(rows * K + 1, generator=g).to(DEV)[1:].view(rows, K)
    if kind == "batched":  # 3-D with a batch stride that does not continue the row pitch
        return torch.randn(3, rows // 3 + 5, K, generator=g).to(DEV)[:, :rows // 3]
    x = torch.randn(rows, K, generator=g)
    if kind == "cpu":
        return x
    return x.to(DEV, {"f64": torch.float64, "f16": torch.float16, "bf16": torch.bfloat16}.get(kind, dtype))


@pytest.mark.gpu
def test_routes(gemm, monkeypatch):
    """Every case of the route table runs exactly the predicted entry point."""
    g = torch.Generator().manual_seed(19)
    torch.backends.cuda.matmul.allow_tf32 = False
    calls = []
    for name in ENTRY:
        orig = getattr(gemm.cabi, name)

        def rec(*a, _orig=orig, _name=name, **kw):
            if _name != "split_tf32" or not kw.get("layout_b", False):  # not the weight's cached split
                calls.append((_name, kw.get("chunk")))
            return _orig(*a, **kw)
        monkeypatch.setattr(gemm.cabi, name, rec)
    lin = torch.nn.functional.linear

    def rec_linear(*a, **kw):
        calls.append(("F.linear", torch.backends.cuda.matmul.allow_tf32))
        return lin(*a, **kw)
    monkeypatch.setattr(torch.nn.functional, "linear", rec_linear)
    monkeypatch.setattr(gemm, "_orig_linear", rec_linear)
    for case in ROUTE_CASES:
        mode, own, long_k, persistent, rows, K, N, kind, train = case
        gemm.MODE, gemm.OWN_KERNEL, gemm.LONG_K_PRESPLIT, gemm.PRESPLIT_PERSISTENT = mode, own, long_k, persistent
        x = _layout(kind, rows, K, g)
        w = torch.randn(N, K, generator=g).to(x.device, x.dtype) / K ** 0.5
        route = _route_of(case)
        calls.clear()
        if train:
            xg = x.detach().requires_grad_(True)
            gemm.linear_train(xg, w).sum().backward()
        else:
            gemm.linear(x, w)
        names = [c[0] for c in calls]
        got = {"T1": ["gemm_f16x3_scaled", "gemm_f16x3_scaled"], "T2": ["gemm_f16x3_scaled"], "T3": ["F.linear"],
               "L0": ["F.linear"], "L1": ["gemm_f16x3_pre"], "L2": ["gemm_3xtf32_pre"], "L3": ["gemm_3xtf32"],
               "L4": ["gemm_3xtf32_raw"], "L5": ["split_tf32", "F.linear"], "L6": ["split_tf32", "F.linear"],
               "L7": ["F.linear"]}[route]
        assert names == got, (case, route, calls)
        if route in ("L5", "L6"):
            assert (calls[0][1] == K) == (route == "L5") and calls[1][1] is True, (case, calls)
        if route in ("L0", "L7", "T3"):
            assert calls[0][1] == (route == "L7"), (case, calls)


MODES = ("auto", "tcgen05", "3xtf32", "fp32", "tf32")
LAYOUTS = ("contiguous", "transposed", "odd_pitch", "misaligned", "batched")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_linear_dropin_layouts(gemm, mode):
    """Every input F.linear takes works in every mode: transposed, odd-pitch, misaligned and batched x, 0 and 1 rows, a
    non-contiguous bias or none, fp16 / bf16 / fp64, CPU tensors.  fp32 CUDA results are within the mode's bound of
    float64 and bit-identical to the same route on an aligned contiguous copy; the rest equals F.linear."""
    gemm.MODE = mode
    g = torch.Generator().manual_seed(20)
    for K, N in ((64, 96), (96, 91)):
        w = make_w("randn", N, K, g).to(DEV)
        b_nc = torch.randn(N, 3, generator=g).to(DEV)[:, 1]
        for rows in (SMALL_M + 6, 1, 0):
            for kind in LAYOUTS if rows > 1 else ("contiguous",):
                x = _layout(kind, rows, K, g)
                for b, act in ((b_nc, 0), (None, 1), (b_nc, 2)):
                    y = gemm.linear(x, w, b, input_act={0: None, 1: "relu", 2: "gelu"}[act])
                    assert y.shape == (*x.shape[:-1], N)
                    want = gemm.linear(x.contiguous().clone(), w, None if b is None else b.contiguous(),
                                       input_act={0: None, 1: "relu", 2: "gelu"}[act])
                    route = predict_route(mode, "f16x3", False, True, rows, K, N)
                    if route not in ("L0", "L7"):  # the project's kernels: layout-blind bit for bit
                        assert torch.equal(y, want), (mode, K, rows, kind, act)
                    if rows:
                        c, unit = {"L0": (C_FP32, U), "L7": (C_TF32_1, 2.0 ** -11), "L1": (C_F16, U), "L2": (C_TF32, U),
                                   "L5": (C_SPLIT, U)}[route]
                        ref, S = ref_and_scale(x.reshape(-1, K), w, b, act)
                        err = (y.reshape(-1, N).double() - ref).abs()
                        floor = 2.0 ** -29 * w.double().abs().sum(1) if route == "L1" else 0.0
                        _observe(f"linear_{route}", err, unit * S, floor)
                        assert (err <= c * unit * S + floor).all(), (mode, K, rows, kind, act)
        for kind in ("f16", "bf16", "f64", "cpu"):
            x = _layout(kind, SMALL_M + 6, K, g)
            wk, bk = w.to(x.device, x.dtype), b_nc.to(x.device, x.dtype)
            assert torch.equal(gemm.linear(x, wk, bk), F.linear(x, wk, bk)), (mode, kind)
            assert torch.equal(gemm.linear_train(x, wk, bk), F.linear(x, wk, bk)), (mode, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [128, 91])
def test_linear_train_layouts_and_scales(gemm, cabi, N):
    """linear_train (T1 at N = 128, T2 at N = 91) with contiguous, misaligned and transposed x: forward, dx, dW and db
    within their bounds of float64 autograd, at gradient scales 1, 1e-12 and 1e-20 (the last two near the +-60 clamp of
    pow2_scale's exponent: the fp16 floor of dy's scale is part of dx's bound), and the same bits for every layout."""
    g = torch.Generator().manual_seed(21)
    M, K = SMALL_M + 100, 64
    w, b = make_w("randn", N, K, g).to(DEV), torch.randn(N, generator=g).to(DEV)
    x0 = torch.randn(M, K, generator=g).to(DEV)
    dy0 = torch.randn(M, N, generator=g).to(DEV)
    for scale in (1.0, 1e-12, 1e-20):
        dy = dy0 * scale
        results = []
        for kind in ("contiguous", "misaligned", "transposed"):
            if kind == "contiguous":
                leaf = x0.clone().requires_grad_(True)
                x = leaf
            elif kind == "misaligned":
                buf = torch.empty(M * K + 1, device=DEV)
                buf[1:] = x0.flatten()
                leaf = buf.requires_grad_(True)
                x = leaf[1:].view(M, K)
            else:
                leaf = x0.t().contiguous().requires_grad_(True)
                x = leaf.t()
            wg, bg = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
            y = gemm.linear_train(x, wg, bg)
            y.backward(dy)
            dx = leaf.grad[1:].view(M, K) if kind == "misaligned" else leaf.grad.t() if kind == "transposed" else leaf.grad
            results.append((y.detach(), dx, wg.grad, bg.grad))
        for r in results[1:]:  # dW is cuBLAS on the caller's layout of x: bounded below, not bit-identical
            for i in (0, 1, 3):
                assert torch.equal(r[i], results[0][i]), (scale, i)
            check_bound("train_dw", r[2], dy.t(), x0.t(), None, 0, C_FP32)
        y, dx, dw, db = results[0]
        check_bound("train_y", y, x0, w, b, 0, C_F16, 16.0, cabi.split_f16_pair_dev(w)[2].item())
        if N % 64 == 0:
            a_dy = cabi.pow2_scale(dy.contiguous(), 12).item()
            w_t = cabi.pow2_scale(w.contiguous(), 14).item()
            check_bound(f"train_dx_{scale:g}", dx, dy, w.t(), None, 0, C_F16, a_dy, w_t)
        else:
            check_bound("train_dx_cublas", dx, dy, w.t(), None, 0, C_FP32)
        check_bound("train_dw", dw, dy.t(), x0.t(), None, 0, C_FP32)
        ref_db, S_db = dy.double().sum(0), dy.double().abs().sum(0)
        err = (db.double() - ref_db).abs()
        _observe("train_db", err, U * S_db)
        assert (err <= C_FP32 * U * S_db).all()


@pytest.mark.gpu
def test_linear_train_nonfinite_dy(gemm):
    """A NaN or inf in dy reaches the rows of dx it belongs to (gemm_f16x3_scaled with the device scale of dy) and leaves
    every other row of dx bit-identical."""
    g = torch.Generator().manual_seed(22)
    M, K, N, r = SMALL_M + 100, 64, 128, 1000
    x, w, b = torch.randn(M, K, generator=g).to(DEV), make_w("randn", N, K, g).to(DEV), torch.randn(N, generator=g).to(DEV)
    dy0 = torch.randn(M, N, generator=g).to(DEV)
    dy0[r, 5] = 0.1  # not the maximum: dy's device scale comes from the other entries

    def dx_of(dy):
        xg = x.clone().requires_grad_(True)
        gemm.linear_train(xg, w, b).backward(dy)
        return xg.grad
    clean = dx_of(dy0)
    rows = torch.arange(M, device=DEV) != r
    for name, v in NONFINITE.items():
        dy = dy0.clone()
        _poke(dy, (r, 5), v)
        dx = dx_of(dy)
        assert not dx[r].isfinite().any(), name
        assert torch.equal(dx[rows], clean[rows]), name


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["auto", "tcgen05", "3xtf32"])
def test_linear_routes_nonfinite(gemm, mode):
    """The non-finite contract through gemm.linear on every tensor-core route (L1-L6), input activation none / ReLU /
    GELU: NaN (four encodings) and inf at one element of x."""
    g = torch.Generator().manual_seed(23)
    M, N, r, k = SMALL_M + 50, 96, 1500, 9
    settings = {"auto": [("f16x3", False, True, 64), ("f16x3", False, True, 96), ("tf32x3", False, False, 64),
                         ("f16x3", True, True, 1024)],
                "tcgen05": [("f16x3", False, True, 100)], "3xtf32": [("f16x3", False, True, 64), ("f16x3", False, True, 1024)]}
    gemm.MODE = mode
    for own, long_k, persistent, K in settings[mode]:
        gemm.OWN_KERNEL, gemm.LONG_K_PRESPLIT, gemm.PRESPLIT_PERSISTENT = own, long_k, persistent
        x0, w = torch.randn(M, K, generator=g).to(DEV), make_w("randn", N, K, g).to(DEV)
        for act in (None, "relu", "gelu"):
            clean = gemm.linear(x0, w, None, input_act=act)
            for name, v in NONFINITE.items():
                x = x0.clone()
                _poke(x, (r, k), v)
                y = gemm.linear(x, w, None, input_act=act)
                ref = F.linear(_act64(x, {None: 0, "relu": 1, "gelu": 2}[act]), w.double())
                assert torch.equal(y.isfinite(), ref.isfinite()), (mode, own, K, act, name)
                rows = torch.arange(M, device=DEV) != r
                assert torch.equal(y[rows], clean[rows]), (mode, own, K, act, name)
