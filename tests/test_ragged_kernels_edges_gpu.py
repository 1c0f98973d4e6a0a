"""GPU: the kernels behind per-sample lengths (a batch of sequences padded at their ends), at their edges.

Each ragged kernel must give every sample exactly what the plain kernel gives that sample alone, unpadded, and must
not read what the padded rows hold: the attention over keys [0, kv_lens[b]) (`ops.attention(kv_lens=)`), the GroupNorm
+ SiLU over rows [0, lens[b]) (`ops.groupnorm_silu(lens=)`), the prompt mean, the row mask, the row pack of the
predictor's keys and the condition injection with per-sample condition lengths.  The attention is also held to the
fp64 bounds of the attention edge suite (kernel_check.attention_reference), which reject a reference that attends to one key more.
"""
import pytest
import torch

from kernel_check import ATTN_RL2, assert_close, assert_rejects, attention_inputs, attention_reference

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"
LENS = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256]


def _lens(v):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def _garbage(t, g):
    """±1e4 in every element of t (a view), in place."""
    t.copy_(torch.where(torch.rand(t.shape, device=dev, generator=g) < 0.5, -1e4, 1e4).to(t.dtype))


@pytest.mark.parametrize("H", [1, 8])
@pytest.mark.parametrize("Nq", [1, 65, 300])
@pytest.mark.parametrize("Nk", [129, 300, 1024])
def test_attention_ragged(Nk, Nq, H):
    from naturalspeech2_pytorch_b200 import ops
    lens = [v for v in LENS if v < Nk] + [Nk]
    B, inner = len(lens), H * 64
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=Nk + 7 * Nq + H)      # windows of one fused projection
    g = torch.Generator(device=dev).manual_seed(Nk * Nq)
    for b, n in enumerate(lens):
        if n < Nk:   # the first key past the length: score 0 and a large value, so attending to it shows
            k[b, n] = 0.0
            v[b, n] = 64.0
        _garbage(k[b, n + 1:], g)
        _garbage(v[b, n + 1:], g)
    out = torch.full((B, Nq, inner), float("nan"), device=dev, dtype=bf)
    ops.attention(q, k, v, out, heads=H, kv_lens=_lens(lens))
    for b, n in enumerate(lens):
        alone = torch.empty(1, Nq, inner, device=dev, dtype=bf)
        ops.attention(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], alone, heads=H)
        assert torch.equal(out[b:b + 1], alone), (b, n)
        ref = attention_reference(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], d_o[b:b + 1], H, 64 ** -0.5)
        assert_close(out[b:b + 1], ref["o"], ref["b_o"], ATTN_RL2, f"sample {b}, {n} keys")
        if n < Nk:   # attending to one key more (a ±1e4 garbage key) must fail the same bounds
            wrong = attention_reference(q[b:b + 1], k[b:b + 1, :n + 1], v[b:b + 1, :n + 1], d_o[b:b + 1], H, 64 ** -0.5)
            assert_rejects(out[b:b + 1], wrong["o"], ref["b_o"], ATTN_RL2, f"sample {b}, {n} + 1 keys")


@pytest.mark.parametrize("B,H,Nq,Nk", [(2, 8, 300, 1024), (3, 2, 65, 129)])
def test_attention_ragged_full_lengths_match_plain(B, H, Nq, Nk):
    from naturalspeech2_pytorch_b200 import ops
    q, k, v, _ = attention_inputs(B, H, Nq, Nk, seed=3)
    a, p = (torch.empty(B, Nq, H * 64, device=dev, dtype=bf) for _ in range(2))
    ops.attention(q, k, v, a, heads=H, kv_lens=_lens([Nk] * B))
    ops.attention(q, k, v, p, heads=H)
    assert torch.equal(a, p)


@pytest.mark.parametrize("resid", [False, True], ids=["plain", "resid"])
@pytest.mark.parametrize("cpg", [4, 64])
def test_groupnorm_silu_ragged(cpg, resid):
    from naturalspeech2_pytorch_b200 import ops
    G, N = 4, 37
    C, lens = G * cpg, [1, 3, N]
    B = len(lens)
    g = torch.Generator(device=dev).manual_seed(cpg)
    x = torch.randn(B, N, C, device=dev, generator=g) * 3 + 0.5
    r = torch.randn(B, N, C, device=dev, generator=g)
    w = torch.randn(C, device=dev, generator=g)
    bias = torch.randn(C, device=dev, generator=g)
    finite = x.clone()
    for b, n in enumerate(lens):
        x[b, n:] = float("nan")
        r[b, n:] = float("nan")
    f32 = torch.full_like(x, float("nan"))
    h = torch.full(x.shape, float("nan"), device=dev, dtype=bf)
    ops.groupnorm_silu(x, w, bias, G, resid=r if resid else None, out_f32=f32, out_bf16=h, lens=_lens(lens))
    for b, n in enumerate(lens):
        a32 = torch.empty(1, n, C, device=dev)
        abf = torch.empty(1, n, C, device=dev, dtype=bf)
        ops.groupnorm_silu(x[b:b + 1, :n].contiguous(), w, bias, G, resid=r[b:b + 1, :n].contiguous() if resid else None,
                           out_f32=a32, out_bf16=abf)
        assert torch.equal(f32[b, :n], a32[0]) and torch.equal(h[b, :n], abf[0]), (b, n)
        assert int((f32[b, n:] != 0).sum()) == 0 and int((h[b, n:] != 0).sum()) == 0
    # sensitivity: statistics over every row (finite padding) differ from the ragged ones
    full = torch.empty_like(x)
    ops.groupnorm_silu(finite, w, bias, G, out_f32=full)
    ragged = torch.empty_like(x)
    ops.groupnorm_silu(finite, w, bias, G, out_f32=ragged, lens=_lens(lens))
    for b, n in enumerate(lens[:-1]):
        assert not torch.equal(full[b, :n], ragged[b, :n]), b


def test_mean_rows_ragged():
    from naturalspeech2_pytorch_b200 import ops
    B, N, D = 4, 103, 300
    lens = [1, 2, 57, N]
    x = torch.randn(B, N, D, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    for b, n in enumerate(lens):
        x[b, n:] = float("nan")
    out = ops.mean_rows(x, torch.empty(B, D, device=dev), lens=_lens(lens))
    for b, n in enumerate(lens):
        s = torch.zeros(D, device=dev)
        for i in range(n):   # the kernel's order: rows one after another, in fp32
            s = s + x[b, i]
        assert torch.equal(out[b], s / torch.full_like(s, n)), b   # a true division, like the kernel's
        assert torch.equal(out[b:b + 1], ops.mean_rows(x[b:b + 1, :n].contiguous(), torch.empty(1, D, device=dev)))


@pytest.mark.parametrize("dtype", [torch.float32, bf])
def test_mask_rows_strided(dtype):
    from naturalspeech2_pytorch_b200 import ops
    B, N, C = 3, 70, 36
    store = torch.randn(N + 5, B, C + 12, device=dev).to(dtype)
    x = store[:N, :, 4:4 + C].transpose(0, 1)          # row stride B (C + 12), batch stride C + 12
    want = x.clone()
    lens = [0, 1, N]
    for b, n in enumerate(lens):
        want[b, n:] = 0
    before = store.clone()
    ops.mask_rows(x, _lens(lens))
    assert torch.equal(x, want)
    rest = torch.ones_like(store, dtype=torch.bool)
    rest[:N, :, 4:4 + C] = False
    assert torch.equal(store[rest], before[rest])       # nothing outside the view is written
    one = torch.randn(B, N, device=dev)                 # (B, N) viewed as one column per row
    ops.mask_rows(one.view(B, N, 1), _lens([3, 0, 70]))
    assert int((one[0, 3:] != 0).sum()) == 0 and int((one[1] != 0).sum()) == 0 and bool((one[2] != 0).all())


def test_pack_rows():
    from naturalspeech2_pytorch_b200 import ops
    B, Na, Nb, C = 4, 25, 40, 128
    a = torch.randn(B, Na, C, device=dev).to(bf)
    bsrc = torch.randn(B, Nb + 3, C + 64, device=dev).to(bf)[:, :Nb, 64:]   # strided window
    la, lb = [1, 25, 7, 25], [40, 1, 13, 0]
    out = torch.full((B, Na + Nb + 5, C), float("nan"), device=dev, dtype=bf)
    ops.pack_rows(a, _lens(la), bsrc, _lens(lb), out)
    for b in range(B):
        want = torch.zeros(Na + Nb + 5, C, device=dev, dtype=bf)
        want[:la[b] + lb[b]] = torch.cat((a[b, :la[b]], bsrc[b, :lb[b]]))
        assert torch.equal(out[b], want), b


@pytest.mark.parametrize("dropped", [False, True], ids=["cond", "null"])
def test_cond_inject_ragged(dropped):
    from naturalspeech2_pytorch_b200 import ops
    B, N, L, D = 5, 50, 40, 128
    g = torch.Generator(device=dev).manual_seed(9)
    x = torch.randn(B, N, D, device=dev, generator=g)
    cproj = torch.randn(B, L, D, device=dev, generator=g)
    null = torch.randn(D, device=dev, generator=g)
    cl = [0, 1, 39, 40, 70]                           # below, at and above the condition length
    drop = torch.tensor([dropped, False, dropped, dropped, True], device=dev)
    for b, n in enumerate(cl):
        cproj[b, n:] = float("nan")
    out = torch.empty(B, N, D, device=dev, dtype=bf)
    ops.cond_inject(x, cproj, out, drop_mask=drop, null_cond=null, cond_lens=_lens(cl))
    pos = torch.arange(N, device=dev)[:, None]
    for b, n in enumerate(cl):
        c = torch.zeros(N, D, device=dev)
        m = min(n, L)
        c[:m] = null if bool(drop[b]) else cproj[b, :m]
        assert torch.equal(out[b], torch.where(pos < m, x[b] + c, x[b]).to(bf)), b
    plain = torch.empty_like(out)
    ops.cond_inject(x, cproj.nan_to_num(), plain, drop_mask=drop, null_cond=null)
    full = torch.empty_like(out)
    ops.cond_inject(x, cproj.nan_to_num(), full, drop_mask=drop, null_cond=null, cond_lens=_lens([L] * B))
    assert torch.equal(plain, full)


def test_ragged_lengths_rejected_before_launch():
    from naturalspeech2_pytorch_b200 import ops
    B, H, N = 2, 1, 70
    q = torch.zeros(B, N, 64, device=dev, dtype=bf)
    o = torch.empty_like(q)
    x = torch.zeros(B, N, 32, device=dev)
    w = torch.ones(32, device=dev)
    bad = [torch.tensor([1, 2], dtype=torch.int64, device=dev), torch.tensor([1, 2], dtype=torch.int32),
           _lens([1, 2, 3]), _lens([0, 5]), _lens([1, N + 1]), _lens([[1, 2]]), [1, 2]]
    before = ops.launch_count()
    for lens in bad:
        with pytest.raises(ValueError):
            ops.attention(q, q, q, o, heads=H, kv_lens=lens)
        with pytest.raises(ValueError):
            ops.groupnorm_silu(x, w, w, 8, out_f32=x.clone(), lens=lens)
        with pytest.raises(ValueError):
            ops.mean_rows(x, torch.empty(B, 32, device=dev), lens=lens)
    for lens in (_lens([-1, 3]), _lens([1, N + 1]), torch.tensor([1, 2], dtype=torch.int32)):
        with pytest.raises(ValueError):
            ops.mask_rows(x, lens)
        with pytest.raises(ValueError):
            ops.pack_rows(q, lens, q, _lens([1, 1]), torch.empty(B, 2 * N, 64, device=dev, dtype=bf))
    with pytest.raises(ValueError):
        ops.cond_inject(x, x, torch.empty(B, N, 32, device=dev, dtype=bf), cond_lens=_lens([-1, 2]))
    with pytest.raises(ValueError):
        ops.attention(q, q, q, o, heads=H, kv_lens=_lens([1, 2]), dropout=(1, 0, 0.5))
    assert ops.launch_count() == before
