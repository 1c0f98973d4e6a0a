"""GPU: the length-aware GEMM, attention and RMSNorm kernels at their tile edges.

Each batch mixes lengths around the 128-row tiles (1, 63, 64, 127, 128, 129, 255, 256, N - 1, N).  The outputs are
pre-filled with NaN: rows of computed tiles must be bit-identical to the call without lengths, rows of skipped tiles
(for the norm: rows at or past the length) must still hold the NaN sentinel, including the F32 epilogue's in-place
residual.  Lengths all equal to N reproduce the plain call bit for bit.  The masked MSE is bit-identical to the call on the unpadded
sample and within fp32 bounds of float64; its backward is bit-identical to the unpadded one and exact zeros past L_b.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
N = 300
LENS = [1, 63, 64, 127, 128, 129, 255, 256, N - 1, N]
B = len(LENS)
BM = 128


def _lens(v=LENS):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def _computed_rows(n):
    return min(-(-n // BM) * BM, N)


def _check(got, ref, lens, what, rows=_computed_rows):
    for b, n in enumerate(lens):
        r = rows(n)
        assert torch.equal(got[b, :r], ref[b, :r]), (what, b, n)
        assert bool(got[b, r:].isnan().all()), (what, b, n, "skipped rows were written")


def _g(*s, dtype=torch.float32, scale=1.0, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn(*s, device=dev, generator=g) * scale).to(dtype)


def _gemm_cases():
    from naturalspeech2_pytorch_b200 import ops
    D, G = 128, 3
    bf = torch.bfloat16
    return {
        "bf16_n128": lambda: dict(a=_g(B, N, 256, dtype=bf), w=_g(128, 256, dtype=bf, scale=0.05),
                                  out=torch.empty(B, N, 128, device=dev, dtype=bf), n=128, epilogue=ops.EPI_BF16,
                                  bias=_g(128)),
        "bf16_n384_conv3": lambda: dict(a=_g(B, N, 128, dtype=bf), w=_g(384, 384, dtype=bf, scale=0.05),
                                        out=torch.empty(B, N, 384, device=dev, dtype=bf), n=384,
                                        epilogue=ops.EPI_BF16, segs=ops.conv3_segs(128)),
        "bf16_silu": lambda: dict(a=_g(B, N, 128, dtype=bf), w=_g(128, 128, dtype=bf, scale=0.05),
                                  out=torch.empty(B, N, 128, device=dev, dtype=bf), n=128, epilogue=ops.EPI_BF16,
                                  bias=_g(128), flags=ops._lib.NS2_GEMM_FLAG_SILU),
        "f32_resid_n128": lambda: dict(a=_g(B, N, 128, dtype=bf), w=_g(128, 128, dtype=bf, scale=0.05),
                                       out=_g(B, N, 128), n=128, epilogue=ops.EPI_F32, bias=_g(128), resid="out"),
        "f32_resid_n256_conv3": lambda: dict(a=_g(B, N, 256, dtype=bf), w=_g(256, 768, dtype=bf, scale=0.05),
                                             out=_g(B, N, 256), n=256, epilogue=ops.EPI_F32, bias=_g(256),
                                             resid="out", segs=ops.conv3_segs(256)),
        "f32_other_resid": lambda: dict(a=_g(B, N, 128, dtype=bf), w=_g(256, 128, dtype=bf, scale=0.05),
                                        out=torch.empty(B, N, 256, device=dev), n=256, epilogue=ops.EPI_F32,
                                        resid=_g(B, N, 256, seed=3)),
        "geglu": lambda: dict(a=_g(B, N, 128, dtype=bf), w=_g(512, 128, dtype=bf, scale=0.05),
                              out=torch.empty(B, N, 256, device=dev, dtype=bf), n=512, epilogue=ops.EPI_GEGLU,
                              bias=_g(512)),
        "wavenet_groups": lambda: dict(a=_g(B, N, D, dtype=bf), w=_g(G * D, 4 * D, dtype=bf, scale=0.05),
                                       out=torch.empty(B, N, G * D, device=dev, dtype=bf), n=D,
                                       epilogue=ops.EPI_WAVENET, bias=_g(2 * G * D), bias1_off=G * D,
                                       segs=ops.conv3_segs(D) + [(0, 3 * D, D, 0, 1)], film=_g(B, G * 2 * D),
                                       film_group_stride=2 * D, groups=G, b_group_row_stride=D,
                                       out_group_col_stride=D, dil=[1, 2, 4]),
    }


@pytest.mark.parametrize("case", list(_gemm_cases()))
def test_gemm_row_lens(case):
    from naturalspeech2_pytorch_b200 import ops
    kw = _gemm_cases()[case]()
    in_place = kw.get("resid") == "out"
    start = kw["out"]

    def run(lens, out):
        k = dict(kw, out=out)
        if in_place:
            k["resid"] = out
        return ops.gemm(**k, row_lens=lens)

    ref = run(None, start.clone())
    got = start.clone()
    if not in_place:
        got.fill_(float("nan"))
    else:   # the residual rows of skipped tiles: NaN, and they must stay NaN (no reduce-add of the padding)
        for b, n in enumerate(LENS):
            got[b, _computed_rows(n):] = float("nan")
    run(_lens(), got)
    _check(got, ref, LENS, case)
    full = start.clone()
    run(_lens([N] * B), full)
    assert torch.equal(full, ref), case


def test_gemm_row_lens_refuses_large_batches():
    from naturalspeech2_pytorch_b200 import ops
    Bb = ops._lib.NS2_GEMM_ROW_LENS_MAX_BATCHES + 1
    a = torch.zeros(Bb, 8, 64, device=dev, dtype=torch.bfloat16)
    before = ops.launch_count()
    with pytest.raises(ValueError, match="row_lens"):
        ops.gemm(a, torch.zeros(64, 64, device=dev, dtype=torch.bfloat16),
                 torch.empty(Bb, 8, 64, device=dev, dtype=torch.bfloat16), n=64, epilogue=ops.EPI_BF16,
                 row_lens=torch.ones(Bb, dtype=torch.int32, device=dev))
    assert ops.launch_count() == before


@pytest.mark.parametrize("kv", [False, True], ids=["q_lens", "q_and_kv_lens"])
def test_attention_q_lens(kv):
    from naturalspeech2_pytorch_b200 import ops
    H, inner = 2, 128
    q, k, v = (_g(B, N, inner, dtype=torch.bfloat16, seed=s) for s in (4, 5, 6))
    lens = _lens()
    kvl = lens if kv else None
    ref = torch.empty(B, N, inner, device=dev, dtype=torch.bfloat16)
    ref_lse = torch.empty(B, H, N, device=dev)
    ops.attention(q, k, v, ref, heads=H, lse=ref_lse, kv_lens=kvl)
    got = torch.full_like(ref, float("nan"))
    lse = torch.full_like(ref_lse, float("nan"))
    q_pad = q.clone()
    for b, n in enumerate(LENS):   # query rows of skipped tiles are never loaded
        q_pad[b, _computed_rows(n):] = float("nan")
    ops.attention(q_pad, k, v, got, heads=H, lse=lse, kv_lens=kvl, q_lens=lens)
    _check(got, ref, LENS, "out")
    _check(lse.transpose(1, 2), ref_lse.transpose(1, 2), LENS, "lse")
    full = torch.empty_like(ref)
    ops.attention(q, k, v, full, heads=H, kv_lens=kvl, q_lens=_lens([N] * B))
    assert torch.equal(full, ref)
    # cross attention: 32 unpadded keys, padded queries
    kc, vc = k[:, :32].contiguous(), v[:, :32].contiguous()
    ref_c = torch.empty_like(ref)
    ops.attention(q, kc, vc, ref_c, heads=H)
    got_c = torch.full_like(ref, float("nan"))
    ops.attention(q_pad, kc, vc, got_c, heads=H, q_lens=lens)
    _check(got_c, ref_c, LENS, "cross")


@pytest.mark.parametrize("dim", [128, 512])
@pytest.mark.parametrize("film", [False, True])
def test_rmsnorm_film_lens(dim, film):
    from naturalspeech2_pytorch_b200 import ops
    x = _g(B, N, dim, seed=7)
    f = _g(B, 3 * dim, seed=8)[:, dim:] if film else None
    gamma = None if film else _g(dim, seed=9)
    ref = ops.rmsnorm_film(x, torch.empty(B, N, dim, device=dev, dtype=torch.bfloat16), gamma=gamma, film=f)
    x_pad = x.clone()
    for b, n in enumerate(LENS):   # rows past the length are not read
        x_pad[b, n:] = float("nan")
    got = torch.full_like(ref, float("nan"))
    ops.rmsnorm_film(x_pad, got, gamma=gamma, film=f, lens=_lens())
    _check(got, ref, LENS, "rmsnorm", rows=lambda n: n)
    full = torch.empty_like(ref)
    ops.rmsnorm_film(x, full, gamma=gamma, film=f, lens=_lens([N] * B))
    assert torch.equal(full, ref)


def test_rmsnorm_film_lens_streaming_grid():
    """A row count large enough for the streaming kernel (every warp walks several rows, prefetching the next)."""
    from naturalspeech2_pytorch_b200 import ops
    Bs, Ns, dim = 32, 1024, 512
    lens_l = [256 + 24 * b for b in range(Bs)]
    x = _g(Bs, Ns, dim, seed=10)
    f = _g(Bs, 2 * dim, seed=11)
    ref = ops.rmsnorm_film(x, torch.empty(Bs, Ns, dim, device=dev, dtype=torch.bfloat16), film=f)
    got = torch.full_like(ref, float("nan"))
    ops.rmsnorm_film(x, got, film=f, lens=torch.tensor(lens_l, dtype=torch.int32, device=dev))
    for b, n in enumerate(lens_l):
        assert torch.equal(got[b, :n], ref[b, :n]) and bool(got[b, n:].isnan().all()), b


@pytest.mark.parametrize("dim", [128, 512])
def test_mse_rows_and_bwd_lens(dim):
    from naturalspeech2_pytorch_b200 import ops
    pred, target = _g(B, N, dim, seed=12), _g(B, N, dim, seed=13)
    pred_pad = _nan_past(pred)
    lens = _lens()
    rows = ops.mse_rows(pred_pad, target, torch.empty(B, device=dev), lens=lens)
    coef = _g(B, seed=14)
    d = torch.full_like(pred, float("nan"))
    d_bf = torch.full((B, N, dim), float("nan"), device=dev, dtype=torch.bfloat16)
    ops.mse_bwd(pred_pad, target, coef, out_bf=d_bf, out_f32=d, lens=lens)
    for b, n in enumerate(LENS):
        p, t = pred[b:b + 1, :n].contiguous(), target[b:b + 1, :n].contiguous()
        alone = ops.mse_rows(p, t, torch.empty(1, device=dev))
        assert torch.equal(rows[b:b + 1], alone), b
        exact = ((p.double() - t.double()) ** 2).mean()
        assert abs(rows[b].item() - exact.item()) <= 1e-5 * exact.item(), b   # fp32 sum of <= 153600 squares
        a_f, a_bf = torch.empty_like(p), torch.empty(p.shape, device=dev, dtype=torch.bfloat16)
        ops.mse_bwd(p, t, coef[b:b + 1].contiguous(), out_bf=a_bf, out_f32=a_f)
        assert torch.equal(d[b, :n], a_f[0]) and torch.equal(d_bf[b, :n], a_bf[0]), b
        assert int((d[b, n:] != 0).sum()) == 0 and int((d_bf[b, n:] != 0).sum()) == 0, b
    full = ops.mse_rows(pred, target, torch.empty(B, device=dev), lens=_lens([N] * B))
    assert torch.equal(full, ops.mse_rows(pred, target, torch.empty(B, device=dev)))


def _nan_past(t):
    t = t.clone()
    for b, n in enumerate(LENS):
        t[b, n:] = float("nan")
    return t
