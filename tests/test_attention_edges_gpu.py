"""GPU: flash attention forward / backward (`ops.attention`, `ops.attention_bwd`) at their tile edges against a float64
reference of softmax(q k^T scale) v and its gradients on the same bf16 operands.

Tile geometry: the forward runs 128 queries x 128-key tiles per CTA (64 query rows per softmax warpgroup); the backward
runs one 128-key tile per CTA (64 keys per warpgroup) over 64-query tiles.  Keys past kv_len in the last tile are
zero-filled and masked; dQ is summed with fp32 atomics over the key tiles; dK / dV stay in registers.
"""
import pytest
import torch

from kernel_check import (ATTN_RL2, U_F32, assert_close, assert_nan, assert_rejects, attention_inputs,
                          attention_reference)

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"
def _wide(B, N, inner, dtype):
    """NaN-filled (B, N, inner + 64) buffer plus one spare row block: outputs go to its first `inner` columns."""
    store = torch.full((B * N + 64, inner + 64), float("nan"), device=dev, dtype=dtype)
    return store, store[:B * N].view(B, N, inner + 64)


def _run(q, k, v, d_o, H, scale, dq_start=None):
    from naturalspeech2_pytorch_b200 import ops
    B, Nq, inner = q.shape
    Nk = k.shape[1]
    o_store, o_full = _wide(B, Nq, inner, bf)
    lse = torch.full((B, H, Nq), float("nan"), device=dev)
    ops.attention(q, k, v, o_full[..., :inner], heads=H, scale=scale, lse=lse)
    dq = torch.zeros(B, Nq, inner, device=dev) if dq_start is None else dq_start.clone()
    dk_store, dk_full = _wide(B, Nk, inner, bf)
    dv_store, dv_full = _wide(B, Nk, inner, bf)
    ops.attention_bwd(q, k, v, o_full[..., :inner], d_o, lse, dq, dk_full[..., :inner], dv_full[..., :inner],
                      heads=H, scale=scale)
    for name, store, full, n in (("o", o_store, o_full, Nq), ("dk", dk_store, dk_full, Nk), ("dv", dv_store, dv_full, Nk)):
        assert_nan(full[..., inner:], f"{name}: columns past heads*64")
        assert_nan(store[B * n:], f"{name}: rows past the last batch")
    return dict(o=o_full[..., :inner], lse=lse, dq=dq, dk=dk_full[..., :inner], dv=dv_full[..., :inner])


def _check(got, ref, what, dq_start=None):
    assert_close(got["o"], ref["o"], ref["b_o"], ATTN_RL2, f"{what} o")
    assert_close(got["lse"], ref["lse"], ref["b_lse"], ATTN_RL2, f"{what} lse")
    dq = got["dq"].double()
    b_dq = ref["b_dq"]
    if dq_start is not None:   # the call adds into dq_accum: compare the increment (fp32 rounding of the sum)
        dq = dq - dq_start.double()
        b_dq = b_dq + U_F32 * (got["dq"].double().abs() + dq_start.double().abs())
    assert_close(dq, ref["dq"], b_dq, ATTN_RL2, f"{what} dq")
    assert_close(got["dk"], ref["dk"], ref["b_dk"], ATTN_RL2, f"{what} dk")
    assert_close(got["dv"], ref["dv"], ref["b_dv"], ATTN_RL2, f"{what} dv")


SHAPES = [
    (1, 1, 1, 1),         # q_len = kv_len = 1: one valid query row and key in the whole tile
    (1, 2, 1, 300),       # q_len = 1 over three key tiles, the last 44 keys wide
    (2, 4, 64, 129),      # last key tile holds one valid key; the second forward warpgroup has no queries
    (2, 2, 65, 128),      # one full key tile; the second forward warpgroup / second backward query tile has 1 row
    (1, 8, 300, 1),       # kv_len = 1: P = 1, dS = 0 up to rounding
    (2, 8, 256, 32),      # a single key tile, 32 keys wide, under two full query tiles
    (1, 2, 32, 135),      # q_len 32: half of one warpgroup's rows; one full key tile and one 7 keys wide
    (3, 3, 513, 385),     # ragged in both: 5 query tiles (last 1 row), 4 key tiles (last 1 key)
    (2, 8, 1024, 1024),   # the benchmarked shape
]


@pytest.mark.parametrize("scale", [None, 0.05, 0.5], ids=["default", "0.05", "0.5"])
@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_attention_fwd_bwd(B, H, Nq, Nk, scale):
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=B * 1000 + Nq + Nk)
    s = 64 ** -0.5 if scale is None else scale
    # dq_accum starts non-zero: the call must add dQ to it
    dq_start = torch.randn(B, Nq, H * 64, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    got = _run(q, k, v, d_o, H, scale, dq_start=dq_start)
    _check(got, attention_reference(q, k, v, d_o, H, s), f"B{B} H{H} Nq{Nq} Nk{Nk} scale {s:.4g}", dq_start=dq_start)


def test_attention_growing_max_fwd_bwd():
    """The adversarial online-softmax inputs of the forward check also go through the backward."""
    B, H, Nq, Nk = 2, 2, 384, 640
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=4, growing_max=True)
    got = _run(q, k, v, d_o, H, None)
    _check(got, attention_reference(q, k, v, d_o, H, 64 ** -0.5), "growing max")


def test_attention_sensitivity_omit_key_tile():
    """The forward and backward tolerances reject a reference that leaves out key tile 1 of 3 (dK / dV compared on
    the keys both references have)."""
    B, H, Nq, Nk = 2, 4, 64, 300
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=12)
    got = _run(q, k, v, d_o, H, None)
    ref = attention_reference(q, k, v, d_o, H, 64 ** -0.5)
    _check(got, ref, "exact reference")
    wrong = attention_reference(q, k, v, d_o, H, 64 ** -0.5, drop_key_tile=1)
    assert_rejects(got["o"], wrong["o"], ref["b_o"], ATTN_RL2, "o without key tile 1")
    assert_rejects(got["dq"], wrong["dq"], ref["b_dq"], ATTN_RL2, "dq without key tile 1")
    keep = torch.cat([torch.arange(0, 128), torch.arange(256, Nk)]).to(dev)
    for name in ("dk", "dv"):
        assert_rejects(got[name][:, keep], wrong[name], ref["b_" + name][:, keep], ATTN_RL2, f"{name} without key tile 1")


def test_attention_bwd_determinism():
    """dK / dV are register-resident and stored once: bit-identical across runs.  dQ (fp32 atomics) only within
    tolerance of the first run."""
    B, H, Nq, Nk = 2, 4, 513, 385
    q, k, v, d_o = attention_inputs(B, H, Nq, Nk, seed=6)
    a = _run(q, k, v, d_o, H, None)
    b = _run(q, k, v, d_o, H, None)
    assert torch.equal(a["o"], b["o"]) and torch.equal(a["lse"], b["lse"])
    assert torch.equal(a["dk"], b["dk"]) and torch.equal(a["dv"], b["dv"])
    ref = attention_reference(q, k, v, d_o, H, 64 ** -0.5)
    assert_close(b["dq"], a["dq"], 2 * ref["b_dq"], ATTN_RL2, "dq run-to-run")


@pytest.mark.parametrize("dropout", [None, (7, 3, 0.25)], ids=["plain", "dropout"])
@pytest.mark.parametrize("B,H,Nq", [(1, 1, 1), (2, 8, 300)])
def test_attention_bwd_single_key_gives_exact_zero_dq_dk(B, H, Nq, dropout):
    """kv_len = 1: the softmax is the constant 1, so dQ and dK are exactly zero (in float64 too: the cross attention
    over one perceiver latent and a one-frame self-attention give exact-zero weight gradients), while dV = P^T dO."""
    from naturalspeech2_pytorch_b200 import ops
    q, k, v, d_o = attention_inputs(B, H, Nq, 1, seed=21 + Nq)
    inner = H * 64
    o = torch.empty(B, Nq, inner, device=dev, dtype=bf)
    lse = torch.empty(B, H, Nq, device=dev)
    ops.attention(q, k, v, o, heads=H, lse=lse, dropout=dropout)
    dq = torch.zeros(B, Nq, inner, device=dev)
    dk, dv = (torch.full((B, 1, inner), float("nan"), device=dev, dtype=bf) for _ in range(2))
    ops.attention_bwd(q, k, v, o, d_o, lse, dq, dk, dv, heads=H, dropout=dropout)
    assert int((dq != 0).sum()) == 0 and int((dk != 0).sum()) == 0
    assert bool(torch.isfinite(dv).all())
    if dropout is None:
        ref = attention_reference(q, k, v, d_o, H, 64 ** -0.5)
        assert_close(dv, ref["dv"], ref["b_dv"], ATTN_RL2, "dv, one key")
