"""GPU: the key-padding attention backward (`ops.attention_bwd(kv_lens=)`, attn_bwd_kernel<false, true>) against a
float64 reference of each sample's attention over its own keys [0, kv_lens[b]), under the bounds of the attention
edge suite (kernel_check.attention_reference).

Lengths straddle the backward's 128-key tiles and its 64-key warpgroup halves ({1, 63, 64, 65, 127, 128, 129, Nk},
those <= Nk), for self attention (Nq = Nk) and cross attention (Nq != Nk), 1 and 8 heads.  Besides the float64 bounds:
d K / d V rows past a sample's length are exact zeros (a key tile wholly past it writes zeros and exits); d K / d V of
sample b are bit-identical to the plain call on its keys alone; large finite junk in the padded K / V rows changes no
valid bit of o, lse, d K or d V; lengths that cover every key reproduce the plain call's d K / d V bit for bit; and a
length of 1 gives exact-zero d Q and d K, as the plain kernel does at kv_len = 1.
"""
import pytest
import torch

from kernel_check import ATTN_RL2, assert_close, attention_inputs, attention_reference

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"
LENGTHS = (1, 63, 64, 65, 127, 128, 129)


def _lens(vals):
    from naturalspeech2_pytorch_b200 import ops
    return ops.lengths(vals, len(vals), None, device=dev)


def _run(q, k, v, d_o, H, kv_lens=None):
    """o, lse, dq, dk, dv; dk / dv start as NaN, so every row the call leaves unwritten shows."""
    from naturalspeech2_pytorch_b200 import ops
    B, Nq, inner = q.shape
    Nk = k.shape[1]
    o = torch.empty(B, Nq, inner, device=dev, dtype=bf)
    lse = torch.empty(B, H, Nq, device=dev)
    ops.attention(q, k, v, o, heads=H, lse=lse, kv_lens=kv_lens)
    dq = torch.zeros(B, Nq, inner, device=dev)
    dk, dv = (torch.full((B, Nk, inner), float("nan"), device=dev, dtype=bf) for _ in range(2))
    ops.attention_bwd(q, k, v, o, d_o, lse, dq, dk, dv, heads=H, kv_lens=kv_lens)
    return dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv)


@pytest.mark.parametrize("H", [1, 8])
@pytest.mark.parametrize("kind", ["self", "cross"])
@pytest.mark.parametrize("Nk", [100, 1024])
def test_attention_bwd_kv_lens(Nk, kind, H):
    lens = sorted({n for n in LENGTHS if n <= Nk} | {Nk})
    B = len(lens)
    Nq = Nk if kind == "self" else 77
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=Nk + Nq + H)
    kl = _lens(lens)
    got = _run(q, k, v, d_o, H, kl)
    scale = 64 ** -0.5
    for b, n in enumerate(lens):
        what = f"Nk{Nk} {kind} H{H} sample {b} (kv_len {n})"
        ref = attention_reference(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], d_o[b:b + 1], H, scale)
        assert_close(got["o"][b:b + 1], ref["o"], ref["b_o"], ATTN_RL2, f"{what} o")
        assert_close(got["lse"][b:b + 1], ref["lse"], ref["b_lse"], ATTN_RL2, f"{what} lse")
        assert_close(got["dq"][b:b + 1], ref["dq"], ref["b_dq"], ATTN_RL2, f"{what} dq")
        assert_close(got["dk"][b:b + 1, :n], ref["dk"], ref["b_dk"], ATTN_RL2, f"{what} dk")
        assert_close(got["dv"][b:b + 1, :n], ref["dv"], ref["b_dv"], ATTN_RL2, f"{what} dv")
        for name in ("dk", "dv"):   # NaN-initialised: != 0 also catches rows left unwritten
            assert int((got[name][b, n:] != 0).sum()) == 0, (what, name, "padding")
        alone = _run(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], d_o[b:b + 1], H)
        for name in ("o", "lse", "dk", "dv"):
            a, g = alone[name][0], got[name][b]
            assert torch.equal(g[:n] if name in ("dk", "dv") else g, a), (what, name, "alone")
        if n == 1:   # a softmax over one key: dS = 0 exactly
            assert int((got["dq"][b] != 0).sum()) == 0 and int((got["dk"][b] != 0).sum()) == 0, what

    # junk in the padded K / V rows: finite, large, and reaches no valid bit
    kj, vj = k.clone(), v.clone()
    for b, n in enumerate(lens):
        kj[b, n:] = 3.0e4
        vj[b, n:] = -1.0e30
    junk = _run(q, kj, vj, d_o, H, kl)
    for name in ("o", "lse", "dk", "dv"):
        assert torch.equal(junk[name], got[name]), (name, "junk")
    for b, n in enumerate(lens):
        ref = attention_reference(q[b:b + 1], k[b:b + 1, :n], v[b:b + 1, :n], d_o[b:b + 1], H, scale)
        assert_close(junk["dq"][b:b + 1], ref["dq"], ref["b_dq"], ATTN_RL2, f"sample {b} dq with junk keys")

    # lengths that cover every key: the plain call's d K / d V, bit for bit
    full = _run(q, k, v, d_o, H, _lens([Nk] * B))
    plain = _run(q, k, v, d_o, H)
    for name in ("o", "lse", "dk", "dv"):
        assert torch.equal(full[name], plain[name]), (name, "full lengths")


def test_attention_bwd_kv_lens_strided_views():
    """d K / d V written into column windows of one fused buffer (the layout training.attention_backward passes), with
    key tiles past a sample's length: the zero rows stay inside each window."""
    from naturalspeech2_pytorch_b200 import ops
    B, H, Nq, Nk = 3, 2, 70, 300
    inner = H * 64
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=5)
    kl = _lens([1, 129, 300])
    o = torch.empty(B, Nq, inner, device=dev, dtype=bf)
    lse = torch.empty(B, H, Nq, device=dev)
    ops.attention(q, k, v, o, heads=H, lse=lse, kv_lens=kl)
    d_kv = torch.full((B, Nk, 2 * inner + 64), float("nan"), device=dev, dtype=bf)
    dq = torch.zeros(B, Nq, inner, device=dev)
    ops.attention_bwd(q, k, v, o, d_o, lse, dq, d_kv[..., :inner], d_kv[..., inner:2 * inner], heads=H, kv_lens=kl)
    assert bool(torch.isnan(d_kv[..., 2 * inner:]).all()), "columns past the window"
    ref = _run(q, k, v, d_o, H, kl)
    assert torch.equal(d_kv[..., :inner], ref["dk"]) and torch.equal(d_kv[..., inner:2 * inner], ref["dv"])
