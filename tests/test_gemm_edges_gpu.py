"""GPU: the segmented wgmma GEMM (`ops.gemm`, all four epilogues) at its tile edges against a float64 reference.

Tile geometry (csrc/gemm.cu): 128 positions x BN columns per tile, BN = 256 when n >= 256 (always for GEGLU) and 128
otherwise (always for WAVENET); consumer warpgroup w owns rows [64 w, 64 w + 64) of a tile; K runs in 64-wide blocks
through a STAGES-deep smem ring (4 stages at BN 256, 6 at BN 128) shared by all tiles of a persistent CTA.
"""
import math

import pytest
import torch

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_nan, assert_rejects, shifted

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _seg_ref(a, w, segs, dil=1):
    """float64 (acc, sum |a||w|, K) per accumulator id of one group: acc[j] = sum_s shifted(a)[.., seg cols] w[j, ..]."""
    a64, w64 = a.double(), w.double()
    acc, mag, K = {}, {}, {}
    for (ac, bc, kl, sh, ai) in segs:
        xs = shifted(a64[..., ac:ac + kl], sh * dil)
        ww = w64[:, bc:bc + kl]
        acc[ai] = acc.get(ai, 0) + xs @ ww.T
        mag[ai] = mag.get(ai, 0) + xs.abs() @ ww.abs().T
        K[ai] = K.get(ai, 0) + kl
    return acc, mag, K


def _out_buffer(B, N, cols, extra_cols, dtype):
    """NaN-filled storage for a (B, N, cols) output viewed as a column window of (B, N, cols + extra_cols) rows, with
    one spare 128-row tile after the last batch: rows past a_rows and columns past n must stay NaN."""
    store = torch.full((B * N + 128, cols + extra_cols), float("nan"), device=dev, dtype=dtype)
    full = store[:B * N].view(B, N, cols + extra_cols)
    return store, full


def _check_untouched(store, full, B, N, cols, what):
    assert_nan(full[..., cols:], f"{what}: columns past n")
    assert_nan(store[B * N:], f"{what}: rows past the last batch")


def _plain_case(B, N, K, n, *, flags=0, seed=0):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    # a: columns [64, 64 + K) of a NaN-filled wider buffer, so a read outside the window (or past a K tail) shows
    a_full = torch.full((B, N, K + 128), float("nan"), device=dev, dtype=bf)
    a = a_full[..., 64:64 + K]
    a.copy_(torch.randn(B, N, K, device=dev, generator=g) * 0.5)
    w = (torch.randn(n, K, device=dev, generator=g) / math.sqrt(K)).to(bf)
    bias = torch.randn(n, device=dev, generator=g)
    resid = torch.randn(B, N, n, device=dev, generator=g)
    acc, mag, Kt = _seg_ref(a, w, [(0, 0, K, 0, 0)])
    pre, pmag = acc[0] + bias.double(), mag[0] + bias.double().abs()
    silu = bool(flags & 4)
    # silu(x) = x sigmoid(x) has |silu'| <= 1.1: the pre-activation error passes through with that factor
    post = pre * torch.sigmoid(pre) if silu else pre
    emag = (1.1 if silu else 1.0) * acc_eps(Kt[0]) * pmag

    store, full = _out_buffer(B, N, n, 64, bf)
    ops.gemm(a, w, full[..., :n], n=n, epilogue=ops.EPI_BF16, bias=bias, flags=flags)
    # bf16 out: 2^-8 |ref| output rounding + fp32 accumulation 2^-20 sqrt(K) sum|a||w| (kernel_check.acc_eps)
    assert_close(full[..., :n], post, U_BF16 * post.abs() + emag, U_BF16 + acc_eps(Kt[0]), "bf16")
    _check_untouched(store, full, B, N, n, "bf16")
    ref32 = post + resid.double()
    store32, full32 = _out_buffer(B, N, n, 64, torch.float32)
    ops.gemm(a, w, full32[..., :n], n=n, epilogue=ops.EPI_F32, bias=bias, resid=resid, flags=flags)
    # fp32 out: 2^-23 |ref| rounding of the bias / residual adds + the same accumulation term
    assert_close(full32[..., :n], ref32, U_F32 * (ref32.abs() + resid.double().abs()) + emag, acc_eps(Kt[0]) * 4,
                 "f32+resid")
    _check_untouched(store32, full32, B, N, n, "f32")


N_COLS = [
    32,    # BN=128: the only tile is 32 wide
    64,    # BN=128: the only tile is 64 wide
    96,    # BN=128: the only tile is 96 wide
    160,   # BN=128: last tile 32 wide
    224,   # BN=128: last tile 96 wide, largest n below the BN switch
    256,   # BN=256: exactly one full tile (first n with BN=256)
    288,   # BN=256: last tile 32 wide
    320,   # BN=256: last tile 64 wide
    352,   # BN=256: last tile 96 wide
    480,   # BN=256: last tile 224 wide
    1408,  # BN=256: last tile 128 wide (the FFN width)
]
N_ROWS = [
    1,     # a single valid row; warpgroup 2 (rows 64..127) has none
    33,    # warpgroup 2 has no valid rows (N % 128 in 1..64)
    64,    # exactly warpgroup 1's rows
    65,    # warpgroup 2 has one valid row
    127,   # one row short of a full tile
    129,   # second tile holds one row
    200,   # second tile: warpgroup 2 holds 8 rows
]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", N_ROWS)
@pytest.mark.parametrize("n", N_COLS)
def test_gemm_plain_tile_edges(n, N, B):
    _plain_case(B, N, 192, n, seed=n * 1000 + N * 10 + B)


@pytest.mark.parametrize("K,n", [
    (80, 96),     # one full 64-block + a 16-wide tail, BN=128
    (80, 288),    # same tail, BN=256 with a 32-wide last tile
    (200, 160),   # 3 blocks + an 8-wide tail
    (1000, 288),  # 15 blocks + a 40-wide tail
])
def test_gemm_k_tail(K, n):
    # a segment that ends at the last column of A and B may have k_len % 64 != 0 (TMA zero-fills the tail block)
    _plain_case(2, 65, K, n, seed=K + n)


@pytest.mark.parametrize("n,N", [
    (160, 129),   # BN=128, 32-wide last tile, one row in the second tile
    (288, 129),   # BN=256, 32-wide last tile
    (1408, 33),   # BN=256, warpgroup 2 empty
])
def test_gemm_silu_epilogue(n, N):
    _plain_case(2, N, 256, n, flags=4, seed=n + N)   # NS2_GEMM_FLAG_SILU, BF16 and F32 + resid


def test_gemm_sensitivity_drop_k_slice():
    """The bf16 and f32 tolerances reject a reference that misses one 16-wide K slice (one wgmma k-step)."""
    from naturalspeech2_pytorch_b200 import ops
    B, N, K, n = 2, 129, 1000, 288
    g = _gen(7)
    a = (torch.randn(B, N, K, device=dev, generator=g) * 0.5).to(bf)
    w = (torch.randn(n, K, device=dev, generator=g) / math.sqrt(K)).to(bf)
    acc, mag, _ = _seg_ref(a, w, [(0, 0, K, 0, 0)])
    out = torch.empty(B, N, n, device=dev, dtype=bf)
    ops.gemm(a, w, out, n=n, epilogue=ops.EPI_BF16)
    bound = U_BF16 * acc[0].abs() + acc_eps(K) * mag[0]
    rl2 = U_BF16 + acc_eps(K)
    assert_close(out, acc[0], bound, rl2, "exact reference")
    k0 = 512
    wrong = acc[0] - a[..., k0:k0 + 16].double() @ w[:, k0:k0 + 16].double().T
    assert_rejects(out, wrong, bound, rl2, "reference without K slice 512..527")
    out32 = torch.empty(B, N, n, device=dev)
    ops.gemm(a, w, out32, n=n, epilogue=ops.EPI_F32)
    b32 = U_F32 * acc[0].abs() + acc_eps(K) * mag[0]
    assert_close(out32, acc[0], b32, acc_eps(K) * 4, "exact reference f32")
    assert_rejects(out32, wrong, b32, acc_eps(K) * 4, "f32 reference without K slice 512..527")


# ----------------------------------------------------------------------------------------------------------------
# convolutions: shifted segments
# ----------------------------------------------------------------------------------------------------------------
def _conv_case(B, N, C, O, segs, dil, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    x = (torch.randn(B, N, C, device=dev, generator=g) * 0.5).to(bf)
    ktot = sum(s[2] for s in segs)
    w = (torch.randn(O, ktot, device=dev, generator=g) / math.sqrt(ktot)).to(bf)
    bias = torch.randn(O, device=dev, generator=g)
    acc, mag, K = _seg_ref(x, w, segs, dil)
    ref, rmag = acc[0] + bias.double(), mag[0] + bias.double().abs()
    store, full = _out_buffer(B, N, O, 32, bf)
    ops.gemm(x, w, full[..., :O], n=O, epilogue=ops.EPI_BF16, bias=bias, segs=segs, dil=[dil])
    bound = U_BF16 * ref.abs() + acc_eps(K[0]) * rmag
    assert_close(full[..., :O], ref, bound, U_BF16 + acc_eps(K[0]), f"conv dil={dil}")
    _check_untouched(store, full, B, N, O, "conv")
    return x, w, bias, full[..., :O].clone(), bound


@pytest.mark.parametrize("N,dil,dgrad", [
    pytest.param(300, 80, False, id="300-80"),     # tap 0 shift 160: more than one 128-row tile
    pytest.param(300, 130, False, id="300-130"),   # tap 0 shift 260, tap 1 shift 130: both cross a tile boundary
    pytest.param(100, 64, False, id="100-64"),     # tap 0 shift 128 >= N: tap 0 reads only zero-filled rows
    pytest.param(100, 200, False, id="100-200"),   # taps 0 and 1 (shifts 400, 200) both beyond the sequence
    pytest.param(65, 1, False, id="65-1"),         # ordinary dil, warpgroup 2 holds one row
    # the causal conv's input gradient (conv_dgrad_segs): shifts 0, -dil, -2 dil read rows after the output position
    pytest.param(300, 4, True, id="dgrad-300-4"),      # the Wavenet backward's shape class
    pytest.param(300, 130, True, id="dgrad-300-130"),  # taps 0 and 1 (shifts -260, -130) cross tile boundaries
    pytest.param(100, 64, True, id="dgrad-100-64"),    # tap 0 shift -128: reaches past the sequence end, reads only zeros
])
def test_gemm_conv3_long_shifts(N, dil, dgrad):
    from naturalspeech2_pytorch_b200 import ops
    segs = ops.conv_dgrad_segs(128, 3, 2) if dgrad else ops.conv3_segs(128)
    _conv_case(2, N, 128, 256, segs, dil, seed=N + dil + (7 if dgrad else 0))


def test_gemm_conv_sensitivity_tap_shift():
    """The conv tolerance rejects a reference whose tap 1 is shifted by one extra row."""
    from naturalspeech2_pytorch_b200 import ops
    segs = ops.conv3_segs(128)
    x, w, bias, out, bound = _conv_case(2, 300, 128, 256, segs, 4, seed=11)
    wrong_segs = [segs[0], (segs[1][0], segs[1][1], segs[1][2], segs[1][3] + 1, 0), segs[2]]
    acc, _, _ = _seg_ref(x, w, wrong_segs, 4)
    assert_rejects(out, acc[0] + bias.double(), bound, U_BF16 + acc_eps(384), "tap 1 shifted by one row")


# ----------------------------------------------------------------------------------------------------------------
# persistent schedule
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", [
    2,    # 64 tiles per CTA: the smem ring wraps dozens of times inside one CTA
    16,   # 8 tiles per CTA, more than STAGES = 4
])
@pytest.mark.parametrize("kind", [
    "linear",   # one 64-wide K block per tile: every tile is a single ring slot
    "conv9",    # 9 segments (NS2_GEMM_MAX_SEGS path), shifts +4..-4: the ring phase wraps inside and across tiles
])
def test_gemm_persistent_ring_wraps(kind, sms):
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200.encoders import _conv_segs
    B, N, C, n = 8, 2048, 64, 256
    segs = [(0, 0, C, 0, 0)] if kind == "linear" else _conv_segs(C, 9, 4)
    prev = ops.set_sm_limit(sms)
    try:
        x, w, bias, out, _ = _conv_case(B, N, C, n, segs, 1, seed=sms)
        again = torch.full_like(out, float("nan"))
        ops.gemm(x, w, again, n=n, epilogue=ops.EPI_BF16, bias=bias, segs=segs, dil=[1])
    finally:
        ops.set_sm_limit(prev)
    assert torch.equal(again, out), "two identical launches differ (the forward GEMM has no atomics)"


def test_gemm_deterministic():
    """Two identical launches of a many-tile problem on all SMs give bit-identical output."""
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(5)
    a = (torch.randn(4, 1000, 512, device=dev, generator=g) * 0.5).to(bf)
    w = (torch.randn(1408, 512, device=dev, generator=g) / 22).to(bf)
    outs = []
    for _ in range(2):
        o = torch.empty(4, 1000, 1408, device=dev)
        ops.gemm(a, w, o, n=1408, epilogue=ops.EPI_F32)
        outs.append(o)
    assert torch.equal(outs[0], outs[1])


# ----------------------------------------------------------------------------------------------------------------
# GEGLU
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,Di", [
    (200, 64),    # half of the first value tile is padding
    (200, 128),   # exactly one value/gate tile pair
    (200, 129),   # second tile pair holds one real column
    (129, 1365),  # the model's FFN width (11 tile pairs, 43 pad columns)
    (1, 341),     # a single row
])
def test_gemm_geglu(N, Di):
    from naturalspeech2_pytorch_b200 import ops
    B, D = 2, 256
    Dp = (Di + 127) // 128 * 128
    g = _gen(Di + N)
    x = (torch.randn(B, N, D, device=dev, generator=g) * 0.7).to(bf)
    W = (torch.randn(2 * Di, D, device=dev, generator=g) / math.sqrt(D)).to(bf)
    b = torch.randn(2 * Di, device=dev, generator=g)
    Wv = torch.zeros(Dp, D, device=dev, dtype=bf); Wv[:Di] = W[:Di]
    Wg = torch.zeros(Dp, D, device=dev, dtype=bf); Wg[:Di] = W[Di:]
    bv = torch.zeros(Dp, device=dev); bv[:Di] = b[:Di]
    bg = torch.zeros(Dp, device=dev); bg[:Di] = b[Di:]
    Wp = torch.stack((Wv.view(-1, 128, D), Wg.view(-1, 128, D)), dim=1).reshape(2 * Dp, D).contiguous()
    bp = torch.stack((bv.view(-1, 128), bg.view(-1, 128)), dim=1).reshape(2 * Dp).contiguous()
    store, full = _out_buffer(B, N, Dp, 32, bf)
    ops.gemm(x, Wp, full[..., :Dp], n=2 * Dp, epilogue=ops.EPI_GEGLU, bias=bp)
    acc, mag, K = _seg_ref(x, W, [(0, 0, D, 0, 0)])
    h = acc[0] + b.double()
    hm = mag[0] + b.double().abs()
    hv, hg, mv, mg = h[..., :Di], h[..., Di:], hm[..., :Di], hm[..., Di:]
    gel = torch.nn.functional.gelu(hg)
    ref = gel * hv
    # out = gelu(g) v: |gelu'| <= 1.13 carries the gate's accumulation error, |gelu(g)| the value's; + bf16 rounding
    bound = U_BF16 * ref.abs() + acc_eps(K[0]) * (1.13 * mg * hv.abs() + gel.abs() * mv)
    assert_close(full[..., :Di], ref, bound, U_BF16 + acc_eps(K[0]), f"geglu Di={Di}")
    assert torch.equal(full[..., Di:Dp], torch.zeros_like(full[..., Di:Dp])), "padded GEGLU columns must be exactly 0"
    _check_untouched(store, full, B, N, Dp, "geglu")


# ----------------------------------------------------------------------------------------------------------------
# WAVENET block: tanh(z) sigmoid(z) + res_conv, z = (dilated conv + b) * gamma + beta
# ----------------------------------------------------------------------------------------------------------------
def _wavenet(B, N, D, G, *, film_scale=1.0, seed=0, strided_film=False, tap_shift_error=False):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    dils = [2 ** i for i in range(G)]
    x = (torch.randn(B, N, G * D, device=dev, generator=g) * 0.5).to(bf)
    wc = (torch.randn(G, D, 3 * D, device=dev, generator=g) / math.sqrt(3 * D)).to(bf)   # taps at [t*D, (t+1)*D)
    wr = (torch.randn(G, D, D, device=dev, generator=g) / math.sqrt(D)).to(bf)
    bc, br = torch.randn(G, D, device=dev, generator=g), torch.randn(G, D, device=dev, generator=g)
    fgs = 2 * D + 32 if strided_film else 2 * D        # film_group_stride
    fbs = G * fgs + 64 if strided_film else G * fgs    # film batch stride
    film_full = torch.full((B, fbs), float("nan"), device=dev)   # gaps between the [gamma | beta] groups stay NaN
    for gi in range(G):
        film_full[:, gi * fgs:gi * fgs + D] = torch.randn(B, D, device=dev, generator=g) * film_scale
        film_full[:, gi * fgs + D:gi * fgs + 2 * D] = torch.randn(B, D, device=dev, generator=g) * film_scale
    wp = torch.cat([wc, wr], dim=2).reshape(G * D, 4 * D).contiguous()
    bias = torch.cat([bc.reshape(-1), br.reshape(-1)]).contiguous()
    segs = ops.conv3_segs(D) + [(0, 3 * D, D, 0, 1)]
    store, full = _out_buffer(B, N, G * D, 64, bf)
    ops.gemm(x, wp, full[..., :G * D], n=D, epilogue=ops.EPI_WAVENET, bias=bias, bias1_off=G * D, segs=segs,
             film=film_full[:, :G * fgs], film_group_stride=fgs, groups=G, a_group_col_stride=D,
             b_group_row_stride=D, out_group_col_stride=D, dil=dils)
    refs, bounds = [], []
    ref_segs = segs
    if tap_shift_error:
        ref_segs = [(s[0], s[1], s[2], s[3] + (1 if i == 0 else 0), s[4]) for i, s in enumerate(segs)]
    for gi in range(G):
        acc, mag, K = _seg_ref(x[..., gi * D:(gi + 1) * D], wp[gi * D:(gi + 1) * D], ref_segs, dils[gi])
        gm = film_full[:, None, gi * fgs:gi * fgs + D].double()
        bt = film_full[:, None, gi * fgs + D:gi * fgs + 2 * D].double()
        z = (acc[0] + bc[gi].double()) * gm + bt
        res = acc[1] + br[gi].double()
        y = torch.tanh(z) * torch.sigmoid(z) + res
        # |d gate/dz| <= 1 carries |gamma| x the conv's accumulation error; the res conv's own accumulation error;
        # 2^-10 for the one-MUFU gate (tanh.approx, relative error 2^-11, |d gate / d tanh| <= 1.3); bf16 rounding
        bnd = (acc_eps(K[0]) * gm.abs() * (mag[0] + bc[gi].double().abs()) + U_F32 * z.abs()
               + acc_eps(K[1]) * (mag[1] + br[gi].double().abs()) + 2.0 ** -10 + U_BF16 * y.abs())
        refs.append(y)
        bounds.append(bnd)
    ref, bound = torch.cat(refs, dim=-1), torch.cat(bounds, dim=-1)
    return store, full, ref, bound


@pytest.mark.parametrize("G,D", [
    (1, 384),   # one group, three 128-wide n-tiles
    (2, 256),   # two groups of two n-tiles
    (8, 128),   # the model's 8 dilation groups (dil up to 128)
])
@pytest.mark.parametrize("N", [
    33,     # warpgroup 2 has no valid rows; dil >= 32 taps read only padding
    200,    # second tile: warpgroup 2 holds 8 rows
    1024,   # the benchmarked sequence length (8 row tiles)
    4096,   # 192-512 tiles: persistent CTAs carry the ring and both accumulators across tiles
])
def test_gemm_wavenet(G, D, N):
    store, full, ref, bound = _wavenet(2, N, D, G, seed=G * 10000 + N)
    assert_close(full[..., :G * D], ref, bound, U_BF16 + 2.0 ** -9, f"wavenet G={G} N={N}")
    _check_untouched(store, full, 2, N, G * D, "wavenet")


@pytest.mark.parametrize("strided", [
    False,   # film_group_stride == 2 D, batch stride == table width
    True,    # film_group_stride = 2 D + 32 and a batch stride 64 wider than the table (gaps hold NaN)
])
def test_gemm_wavenet_film_saturation_and_strides(strided):
    # FiLM entries ~ N(0, 10^2): |z| reaches ~30, where the one-MUFU gate must saturate to 0 / 1 cleanly
    store, full, ref, bound = _wavenet(3, 200, 128, 8, film_scale=10.0, seed=3, strided_film=strided)
    assert_close(full[..., :8 * 128], ref, bound, U_BF16 + 2.0 ** -9, "wavenet saturated")
    _check_untouched(store, full, 3, 200, 8 * 128, "wavenet saturated")


def test_gemm_wavenet_sensitivity_tap_shift():
    """The WAVENET tolerance rejects a reference whose tap 0 is shifted by one row."""
    _, full, _, bound = _wavenet(2, 200, 128, 2, seed=9)
    _, _, wrong, _ = _wavenet(2, 200, 128, 2, seed=9, tap_shift_error=True)
    assert_rejects(full[..., :256], wrong, bound, U_BF16 + 2.0 ** -9, "wavenet tap 0 shifted by one row")
