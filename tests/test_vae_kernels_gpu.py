"""GPU: the SD-VAE glue kernels of csrc/vae.cu (GroupNorm statistics, the fused im2col, the AttnBlock row softmax,
post_quant_conv, the NCHW conversion) each against a float64 torch restatement of the same operation, at the shapes
`generate.py` and `extract_latent.py` run (256- and 512-px images: 1024- and 4096-column softmax, GroupNorm over up to
262 144 pixels, im2col grids at the 132 * 16 block cap) and at the edges where the kernels go wrong (offset and constant
GroupNorm groups, ragged tails, odd sizes, the zero padding columns, argument rejection); then both halves of the
autoencoder end to end at production size against the fp32 oracle."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MDT_ERR_ARG = -1
EPS = 1e-6                     # Normalize's GroupNorm eps (autoencoder.py:34-35), the one mdt_vae_im2col applies


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    """The fp32 references (the oracle decode / encode, the attention-score products) run without TF32."""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def ops():
    from maskdit_b200 import ops as o
    return o


def cuda_gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def bf16_ulp(t):
    """Spacing of bf16 numbers at |t| (float64 tensor): 2^(e - 7) for |t| in [2^e, 2^(e+1))."""
    e = torch.floor(torch.log2(t.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


# ---- GroupNorm(32) statistics ----------------------------------------------------------------------------------------
# Group content (mean, sigma), or ("c", value) for an exactly constant group.  offset / sigma reaches 3000, where the
# one-pass fp32 variance cancels, and the constants are non-dyadic so that n * v * v is not exact in any precision.
KINDS = [(0.0, 1.0), (30.0, 1.0), (300.0, 1.0), (3000.0, 1.0), ("c", 7.3), ("c", 123.456), ("c", -0.1), (-750.0, 0.25)]


def grouped_input(B, P, C, seed, layout):
    """x [B, P, C] f32 on the GPU; const [B, 32] bool.  layout "mixed": group (b, g) is KINDS[(g + 3b) % 8];
    "one_constant": every group N(0.5, 2) but (b=0, g=5), which is the constant 123.456."""
    cg = C // 32
    x = torch.randn(B, P, 32, cg, generator=cuda_gen(seed), device="cuda")
    const = torch.zeros(B, 32, dtype=torch.bool)
    for b in range(B):
        for g in range(32):
            if layout == "mixed":
                kind = KINDS[(g + 3 * b) % len(KINDS)]
            else:
                kind = ("c", 123.456) if (b, g) == (0, 5) else (0.5, 2.0)
            if kind[0] == "c":
                x[b, :, g] = kind[1]
                const[b, g] = True
            else:
                x[b, :, g] = x[b, :, g] * kind[1] + kind[0]
    return x.reshape(B, P, C).contiguous(), const


def gn_stats(x, B, P, C):
    """mdt_vae_gn_stats exactly as vae.py::_gn_stats calls it."""
    o = ops()
    sums = torch.empty(B, 32, 2, dtype=torch.float64, device="cuda")
    scratch = torch.empty(B * ((P + 255) // 256) * 64, dtype=torch.float32, device="cuda")
    o.check(o.lib().mdt_vae_gn_stats(o.ptr(x), o.ptr(sums), o.ptr(scratch), B, P, C, o.stream_ptr()),
            "mdt_vae_gn_stats")
    return sums


def gn_ref(x, B, P, C):
    """Two-pass float64 group mean and (biased) variance [B, 32]."""
    x64 = x.double().view(B, P, 32, C // 32)
    m = x64.mean(dim=(1, 3))
    v = (x64 - m[:, None, :, None]).square().mean(dim=(1, 3))
    return m, v


@pytest.mark.parametrize("layout", ["mixed", "one_constant"])
@pytest.mark.parametrize("P", [35, 256, 1089, 65536])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("C", [128, 256, 512])
def test_gn_stats_vs_float64(C, B, P, layout):
    """P = 35: one ragged chunk; 256: exactly one chunk; 1089 (33^2): ragged last of five; 65536: 256 chunks.
    Mean and variance are derived from the returned sums as mdt_vae_im2col derives them (fp64 quotients, the mean and
    the variance cast to float, the variance clamped at 0)."""
    x, const = grouped_input(B, P, C, seed=C + 7 * B + P, layout=layout)
    sums = gn_stats(x, B, P, C)
    assert torch.equal(gn_stats(x, B, P, C), sums), "GroupNorm statistics differ between two runs"
    cnt = float(P * (C // 32))
    m = sums[..., 0] / cnt
    raw = sums[..., 1] / cnt - m * m                                   # the one-pass variance before the cast
    mean_k = m.float().double()
    var_k = raw.float().double().clamp_min(0.0)
    m_ref, v_ref = gn_ref(x, B, P, C)
    const = const.cuda()
    assert torch.isfinite(sums).all() and torch.isfinite(raw).all()
    err_m = (mean_k - m_ref).abs() / (m_ref.abs() + v_ref.sqrt())
    err_v = torch.where(const, torch.zeros_like(v_ref), (var_k - v_ref).abs() / v_ref)
    # a constant group's one-pass variance is 0 up to the fp64 rounding of n * v^2 (what the clamp absorbs)
    const_raw = torch.where(const, raw.abs() / m_ref.square(), torch.zeros_like(raw))
    print(f"C={C} B={B} P={P} {layout}: worst mean error {err_m.max().item():.2e} (|mean| + sigma), "
          f"variance {err_v.max().item():.2e} (rel), constant-group raw variance {const_raw.max().item():.2e} (mean^2)")
    assert err_m.max().item() <= 1e-6, (err_m.max().item(), torch.nonzero(err_m > 1e-6)[:4].tolist())
    assert err_v.max().item() <= 1e-5, (err_v.max().item(), torch.nonzero(err_v > 1e-5)[:4].tolist())
    assert const_raw.max().item() <= 1e-14, const_raw.max().item()


# ---- fused im2col -----------------------------------------------------------------------------------------------------
def im2col(src, sums, gamma, beta, silu, ks, up, B, H, W, C, Kp, fill=7.0):
    """mdt_vae_im2col exactly as vae.py::_conv calls it, into a buffer pre-filled with `fill`."""
    o = ops()
    A = torch.full((B * H * W, Kp), fill, dtype=torch.bfloat16, device="cuda")
    o.check(o.lib().mdt_vae_im2col(o.ptr(src), o.ptr(sums), o.ptr(gamma), o.ptr(beta), int(silu), ks, up, o.ptr(A),
                                   B, H, W, C, Kp, o.stream_ptr()), "mdt_vae_im2col")
    return A


def im2col_ref(src, gamma, beta, norm, silu, ks, up, B, H, W, C):
    """float64: GroupNorm(32, eps 1e-6) -> swish -> nearest 2x -> unfold, laid out [(b, y, x), (ky, kx, c)]."""
    x = src.double().view(B, H // up, W // up, C).permute(0, 3, 1, 2)
    if norm:
        x = F.group_norm(x, 32, gamma.double(), beta.double(), eps=EPS)
    if silu:
        x = x * torch.sigmoid(x)
    if up == 2:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    u = F.unfold(x, kernel_size=ks, padding=ks // 2)                   # [B, C*ks*ks, H*W], (c, ky, kx)
    return u.view(B, C, ks, ks, H * W).permute(0, 4, 2, 3, 1).reshape(B * H * W, ks * ks * C)


# (C, B, H, W) of the output; up = 2 only where H and W are even.  C = 512 at 64x64 with B = 2 (8192 pixels, 2 per
# block) and C = 128 at 256x256 (65536 pixels, 8 per block) launch more than 132 * 16 blocks, so every block walks
# several pixels in the grid-stride loop.
IM2COL_SHAPES = [(4, 2, 5, 7), (4, 2, 8, 10), (128, 3, 5, 7), (128, 3, 6, 10), (256, 2, 16, 12), (512, 2, 64, 64),
                 (128, 1, 256, 256)]


@pytest.mark.parametrize("C,B,H,W", IM2COL_SHAPES)
def test_im2col_vs_float64(C, B, H, W):
    """Every (ks, up, GroupNorm, swish) combination the kernel serves; each element within one bf16 rounding of the
    float64 value, the padding columns ks*ks*C..Kp exactly zero, constant groups giving bf16(beta) (or its swish)."""
    g = torch.Generator().manual_seed(C * H + W)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).cuda()
    beta = (0.5 * torch.randn(C, generator=g)).cuda()
    worst = {}
    for up in (1, 2):
        if H % up or W % up:
            continue
        Hs, Ws = H // up, W // up
        plain = torch.randn(B, Hs * Ws, C, generator=cuda_gen(C + H + up), device="cuda")
        for norm in ((False, True) if C % 128 == 0 else (False,)):
            if norm:
                src, const = grouped_input(B, Hs * Ws, C, seed=C + H + W + up, layout="mixed")
                sums = gn_stats(src, B, Hs * Ws, C)
            else:
                src, const, sums = plain, None, None
            for silu in (False, True):
                for ks in (1, 3):
                    Kp = (ks * ks * C + 7) // 8 * 8 + 8
                    A = im2col(src, sums, gamma if norm else None, beta if norm else None, silu, ks, up, B, H, W, C,
                               Kp)
                    ref = im2col_ref(src, gamma, beta, norm, silu, ks, up, B, H, W, C)
                    got = A.double()
                    what = f"ks={ks} up={up} norm={norm} silu={silu}"
                    assert torch.isfinite(got).all(), what
                    assert not got[:, ks * ks * C:].any(), f"{what}: nonzero padding column"
                    got = got[:, :ks * ks * C]
                    tol = 2.0 ** -8 * ref.abs() + 1e-6 * ref.abs().max()
                    excess = ((got - ref).abs() / tol).max().item()
                    worst[what] = excess
                    assert excess <= 1.0, (what, excess, torch.nonzero((got - ref).abs() > tol)[:4].tolist())
                    if norm:
                        # constant groups: every in-image element is bf16(beta) (swish(beta)) to one bf16 ulp
                        b_idx, g_idx = torch.nonzero(const, as_tuple=True)
                        cg = C // 32
                        want = beta.double()
                        if silu:
                            want = want * torch.sigmoid(want)
                        for b, gg in zip(b_idx.tolist(), g_idx.tolist()):
                            rows = slice(b * H * W, (b + 1) * H * W)
                            ch = slice(gg * cg, (gg + 1) * cg)
                            centre = got[rows].reshape(H * W, ks * ks, C)[:, (ks * ks) // 2, ch]   # always in the image
                            w = want[ch].to(torch.bfloat16).double()
                            assert ((centre - w).abs() <= bf16_ulp(w)).all(), (what, b, gg)
    print(f"C={C} B={B} {H}x{W}: worst |error| / bound per combination", {k: round(v, 3) for k, v in worst.items()})


def test_im2col_clamps_negative_one_pass_variance():
    """Sums whose one-pass variance q/n - m^2 comes out below zero (the fp64 rounding of n * m^2 of a constant group can
    land on either side of q) must normalise with variance 0: beta (swish(beta)), never rsqrt of a negative number."""
    C, B, H, W = 128, 1, 4, 4
    v = 123.456
    src = torch.full((B, H * W, C), v, device="cuda")
    n, k = H * W * (C // 32), float(np.float32(v))
    sums = torch.empty(B, 32, 2, dtype=torch.float64)
    sums[..., 0] = n * k
    sums[..., 1] = n * k * k - 1e-2 * n                              # q / n - m^2 = -1e-2, far below -eps
    sums = sums.cuda()
    gamma = torch.linspace(0.5, 1.5, C, device="cuda")
    beta = torch.linspace(-2.0, 2.0, C, device="cuda")
    for silu in (0, 1):
        A = im2col(src, sums, gamma, beta, silu, 1, 1, B, H, W, C, C)
        want = beta.double() * torch.sigmoid(beta.double()) if silu else beta.double()
        w = want.to(torch.bfloat16).double()
        assert torch.isfinite(A.double()).all(), f"silu={silu}: non-finite output"
        assert ((A.double() - w).abs() <= bf16_ulp(w)).all(), f"silu={silu}"


# ---- AttnBlock row softmax --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [128, 512])
@pytest.mark.parametrize("rows,cols", [(64, 64), (1024, 1024), (4096, 4096), (1000, 33)])
def test_softmax_rows_vs_float64(rows, cols, c):
    """softmax(c^-1/2 * S) per row into bf16: scaled logits up to +-80 (row r spans +-80 * (r % 5) / 4), one row in 11
    with a single entry at 80, and every seventh row constant at a scaled 120, -120 or 0.37 in turn: a uniform row,
    whatever its common value, since softmax does not see a shift (exp(+-120) is out of fp32 range)."""
    o = ops()
    scale = float(np.float32(c ** -0.5))
    g = cuda_gen(rows + cols + c)
    spread = 80.0 * (torch.arange(rows, device="cuda") % 5).double() / 4
    S = (torch.rand(rows, cols, generator=g, device="cuda", dtype=torch.float64) * 2 - 1) * spread[:, None] / scale
    const_rows = torch.arange(0, rows, 7, device="cuda")
    S[const_rows] = torch.tensor([120.0, -120.0, 0.37], dtype=torch.float64, device="cuda")[const_rows // 7 % 3,
                                                                                            None] / scale
    S[3::11, cols // 2] = 80.0 / scale
    S = S.float().contiguous()
    P = torch.full((rows, cols), 3.0, dtype=torch.bfloat16, device="cuda")
    o.check(o.lib().mdt_vae_softmax_rows(o.ptr(S), scale, o.ptr(P), rows, cols, o.stream_ptr()),
            "mdt_vae_softmax_rows")
    ref = torch.softmax(S.double() * scale, dim=1)
    got = P.double()
    assert torch.isfinite(got).all()
    excess = ((got - ref).abs() / (bf16_ulp(ref) + 1e-6)).max().item()
    row_err = (got.sum(1) - 1).abs().max().item()
    print(f"softmax {rows}x{cols} c={c}: worst |error| / (1 ulp + 1e-6) {excess:.3f}, worst |row sum - 1| {row_err:.2e}")
    assert excess <= 1.0, excess
    assert row_err <= 2.0 ** -7, row_err


# ---- post_quant_conv and the NCHW image -------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 4, 8])
def test_post_quant_vs_float64(C):
    o = ops()
    B, P, sf = 3, 1001, 0.18215
    g = torch.Generator().manual_seed(C)
    z = (torch.randn(B, C, P, generator=g) * sf * 4).cuda()
    W = (torch.randn(C, C, generator=g) * C ** -0.5).cuda()
    bias = (0.05 * torch.randn(C, generator=g)).cuda()
    out = torch.empty(B * P, C, device="cuda")
    o.check(o.lib().mdt_vae_post_quant(o.ptr(z), o.ptr(W), o.ptr(bias), sf, o.ptr(out), B, C, P, o.stream_ptr()),
            "mdt_vae_post_quant")
    want = (z.double().permute(0, 2, 1) / float(np.float32(sf))) @ W.double().t() + bias.double()
    r = ((out.double() - want.reshape(B * P, C)).norm() / want.norm()).item()
    print(f"post_quant C={C}: rel-L2 {r:.2e}")
    assert r <= 1e-6, r


@pytest.mark.parametrize("C,ldx", [(3, 8), (5, 13), (8, 8)])
def test_rows_to_nchw_exact(C, ldx):
    """conv_out's rows (ldx = 8, 3 valid) and other strides: a bit-exact transpose of the first C columns."""
    o = ops()
    B, P = 2, 1001
    x = torch.randn(B * P, ldx, generator=cuda_gen(ldx), device="cuda")
    out = torch.full((B, C, P), 9.0, device="cuda")
    o.check(o.lib().mdt_vae_rows_to_nchw(o.ptr(x), o.ptr(out), B, P, C, ldx, o.stream_ptr()), "mdt_vae_rows_to_nchw")
    assert torch.equal(out, x.view(B, P, ldx)[..., :C].permute(0, 2, 1))


# ---- argument rejection -----------------------------------------------------------------------------------------------
def test_bad_arguments_are_rejected_without_writing():
    o = ops()
    L, sp = o.lib(), o.stream_ptr()
    x = torch.randn(2 * 64 * 512 + 4, device="cuda")
    scratch = torch.zeros(4096, device="cuda")
    sums = torch.full((2, 32, 2), 5.0, dtype=torch.float64, device="cuda")
    gamma, beta = torch.ones(1024, device="cuda"), torch.zeros(1024, device="cuda")
    A = torch.full((2 * 8 * 8 * 9 * 512 + 64,), 3.0, dtype=torch.bfloat16, device="cuda")
    out = torch.full((4096,), 9.0, device="cuda")
    snap = [t.clone() for t in (sums, scratch, A, out)]
    P, H, W = 64, 8, 8
    cases = {
        "gn_stats C=64": lambda: L.mdt_vae_gn_stats(o.ptr(x), o.ptr(sums), o.ptr(scratch), 2, P, 64, sp),
        "gn_stats C=640": lambda: L.mdt_vae_gn_stats(o.ptr(x), o.ptr(sums), o.ptr(scratch), 2, P, 640, sp),
        "gn_stats misaligned x": lambda: L.mdt_vae_gn_stats(o.ptr(x) + 4, o.ptr(sums), o.ptr(scratch), 2, P, 128, sp),
        "im2col Kp % 8": lambda: L.mdt_vae_im2col(o.ptr(x), 0, 0, 0, 0, 3, 1, o.ptr(A), 2, H, W, 128, 9 * 128 + 4,
                                                  sp),
        "im2col Kp < ks*ks*C": lambda: L.mdt_vae_im2col(o.ptr(x), 0, 0, 0, 0, 3, 1, o.ptr(A), 2, H, W, 128,
                                                        9 * 128 - 8, sp),
        "im2col up=2 with stride=2": lambda: L.mdt_vae_im2col_strided(o.ptr(x), 0, 0, 0, 0, 3, 2, 2, 0, o.ptr(A), 2,
                                                                      4, 4, 128, 9 * 128, sp),
        "im2col pad >= ks": lambda: L.mdt_vae_im2col_strided(o.ptr(x), 0, 0, 0, 0, 3, 1, 1, 3, o.ptr(A), 2, H, W, 128,
                                                             9 * 128, sp),
        "im2col H % up": lambda: L.mdt_vae_im2col(o.ptr(x), 0, 0, 0, 0, 3, 2, o.ptr(A), 2, 5, W, 128, 9 * 128, sp),
        "im2col C % 4": lambda: L.mdt_vae_im2col(o.ptr(x), 0, 0, 0, 0, 3, 1, o.ptr(A), 2, H, W, 6, 56, sp),
        "im2col sums without gamma": lambda: L.mdt_vae_im2col(o.ptr(x), o.ptr(sums), 0, o.ptr(beta), 1, 3, 1,
                                                              o.ptr(A), 2, H, W, 128, 9 * 128, sp),
        "im2col sums with C % 128": lambda: L.mdt_vae_im2col(o.ptr(x), o.ptr(sums), o.ptr(gamma), o.ptr(beta), 1, 3,
                                                             1, o.ptr(A), 2, H, W, 64, 9 * 64, sp),
        "im2col misaligned src": lambda: L.mdt_vae_im2col(o.ptr(x) + 4, 0, 0, 0, 0, 3, 1, o.ptr(A), 2, H, W, 128,
                                                          9 * 128, sp),
        "im2col misaligned A": lambda: L.mdt_vae_im2col(o.ptr(x), 0, 0, 0, 0, 3, 1, o.ptr(A) + 8, 2, H, W, 128,
                                                        9 * 128, sp),
        "post_quant C=9": lambda: L.mdt_vae_post_quant(o.ptr(x), o.ptr(x), o.ptr(x), 0.18215, o.ptr(out), 2, 9, 64,
                                                       sp),
        "post_quant scale_factor=0": lambda: L.mdt_vae_post_quant(o.ptr(x), o.ptr(x), o.ptr(x), 0.0, o.ptr(out), 2, 4,
                                                                  64, sp),
        "softmax_rows rows=0": lambda: L.mdt_vae_softmax_rows(o.ptr(x), 0.1, o.ptr(A), 0, 64, sp),
        "rows_to_nchw ldx < C": lambda: L.mdt_vae_rows_to_nchw(o.ptr(x), o.ptr(out), 2, 64, 8, 3, sp),
    }
    for what, call in cases.items():
        assert call() == MDT_ERR_ARG, what
    torch.cuda.synchronize()
    for t, s in zip((sums, scratch, A, out), snap):
        assert torch.equal(t, s), "a rejected call wrote its output"


# ---- both halves end to end at production size ------------------------------------------------------------------------
def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def test_decode_256px_and_512px_vs_fp32_oracle():
    """generate.py's decodes: two 32x32 latents -> 256x256 (1024-column softmax, GroupNorm over 65536 pixels) and one
    64x64 latent -> 512x512 (4096 columns, 262144 pixels), against the fp32 oracle run on the GPU with TF32 off; the
    image is bit-identical when the im2col operands are built 2048 rows at a time."""
    from maskdit_b200.vae import AutoencoderKLDecoder
    from oracle import vae_oracle as VO
    o = ops()
    sd = VO.make_vae_state_dict(3)
    vae = AutoencoderKLDecoder()
    vae.load_state_dict(sd, strict=True)
    vae = vae.cuda().eval()
    sdc = {k: v.cuda() for k, v in sd.items()}
    g = torch.Generator().manual_seed(41)
    for B, h in ((2, 32), (1, 64)):
        z = (torch.randn(B, 4, h, h, generator=g) * 0.18215 * 4.0).cuda()
        vae.max_rows = 1 << 21
        img = vae.decode(z)
        with torch.no_grad():
            ref = VO.decode(sdc, z)
        assert img.shape == ref.shape == (B, 3, 8 * h, 8 * h) and torch.isfinite(img).all()
        r = rel(img, ref)
        diff = (o.to_uint8_nhwc(img.contiguous()).int() - VO.to_uint8(ref).int()).abs().float()
        print(f"decode {8 * h}x{8 * h} (B={B}): rel-L2 vs the fp32 oracle {r:.3e}, 8-bit mean |diff| "
              f"{diff.mean().item():.3f} max {diff.max().item():.0f}")
        assert r <= 1e-2, r
        assert diff.mean().item() <= 1.5
        vae.max_rows = 2048
        assert torch.equal(vae.decode(z), img), "decode changes with the im2col chunking"
        del img, ref, diff
        torch.cuda.empty_cache()


def test_encode_256px_vs_fp32_oracle():
    """extract_latent.py's encode at 256x256 against the fp32 oracle on the GPU with TF32 off."""
    from maskdit_b200.vae import AutoencoderKLEncoder
    from oracle import vae_encode_oracle as VE
    sd = VE.make_vae_encoder_state_dict(4)
    e = AutoencoderKLEncoder()
    e.load_state_dict(sd, strict=True)
    e = e.cuda().eval()
    g = torch.Generator().manual_seed(43)
    base = F.interpolate(torch.rand(1, 3, 32, 32, generator=g), size=256, mode="bilinear", align_corners=False)
    x = (base * 1.6 - 0.8 + 0.2 * torch.rand(1, 3, 256, 256, generator=g)).clamp(-1, 1).cuda()
    m = e.encode_moments(x)
    with torch.no_grad():
        ref = VE.encode_moments({k: v.cuda() for k, v in sd.items()}, x)
    assert m.shape == ref.shape == (1, 8, 32, 32) and torch.isfinite(m).all()
    rm, rl = rel(m[:, :4], ref[:, :4]), rel(m[:, 4:], ref[:, 4:])
    print(f"encode 256x256: rel-L2 vs the fp32 oracle mean {rm:.3e} logvar {rl:.3e}")
    assert rm <= 2e-2 and rl <= 2e-2, (rm, rl)
