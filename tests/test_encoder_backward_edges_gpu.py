"""GPU: the kernels of the conditioning front end's backward pass at their edges against float64 references
(tests/kernel_check.py bounds; NaN-filled regions must stay untouched; one sensitivity test per family).

  ops.wgrad with NEGATIVE shift_units   the "same"-padded k=9 conv taps past the centre read x[n + s] (TMA zero fill
                                        past the end of each sample)
  ops.silu_bwd                          bf16 in / out, including saturated |pre|
  ops.embedding_bwd                     scatter-add with repeated ids, the pad row, rows that never occur
  ops.expand_encodings_bwd              segmented sums over each phoneme's frames (32-frame x 128-channel CTAs)
"""
import pytest
import torch

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_nan, assert_rejects, shifted

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"


# ---------------------------------------------------------------------------------------------------------------
# wgrad, negative shifts
# ---------------------------------------------------------------------------------------------------------------
def _wgrad_neg(B, N, n, k, s, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    dy = torch.randn(B, N, n, device=dev, generator=g).to(bf)
    x = torch.randn(B, N, k, device=dev, generator=g).to(bf)
    dw = torch.full((n + 8, k + 32), float("nan"), device=dev)
    dw[:n, :k] = torch.randn(n, k, device=dev, generator=g)
    start = dw[:n, :k].clone()
    ops.wgrad(dy, x, dw, n=n, k=k, shift_units=s)
    assert_nan(dw[n:], "dW rows past n")
    assert_nan(dw[:, k:], "dW columns past k")
    return dy, x, start, dw[:n, :k]


def _wgrad_ref(dy, x, s):
    xs = shifted(x.double(), s)
    return torch.einsum("bmn,bmk->nk", dy.double(), xs), torch.einsum("bmn,bmk->nk", dy.double().abs(), xs.abs())


def _wgrad_bound(got, start, mag, positions):
    return acc_eps(positions) * mag + U_F32 * (got.double().abs() + start.double().abs())


@pytest.mark.parametrize("N", [65, 300])
@pytest.mark.parametrize("rel", ["-1", "-4", "-(N-1)", "-N", "-(N+37)"])
def test_wgrad_negative_shift(N, rel):
    s = {"-1": -1, "-4": -4, "-(N-1)": -(N - 1), "-N": -N, "-(N+37)": -(N + 37)}[rel]
    B = 2
    dy, x, start, got = _wgrad_neg(B, N, 128, 224, s, seed=N * 100 + len(rel))
    ref, mag = _wgrad_ref(dy, x, s)
    bound = _wgrad_bound(got, start, mag, B * N)
    assert_close(got.double() - start.double(), ref, bound, acc_eps(B * N) * 4, f"N={N} shift={s}")
    if s <= -N:
        assert torch.equal(got, start), "a tap entirely past the end must add exactly zero"


def test_wgrad_negative_shift_sensitivity():
    B, N = 2, 300
    dy, x, start, got = _wgrad_neg(B, N, 128, 224, -4, seed=5)
    _, mag = _wgrad_ref(dy, x, -4)
    wrong, _ = _wgrad_ref(dy, x, -3)
    assert_rejects(got.double() - start.double(), wrong, _wgrad_bound(got, start, mag, B * N), acc_eps(B * N) * 4,
                   "tap shifted by one row")


# ---------------------------------------------------------------------------------------------------------------
# silu_bwd
# ---------------------------------------------------------------------------------------------------------------
def _silu_grad64(x, dy):
    s = torch.sigmoid(x)
    return dy * s * (1 + x * (1 - s))


def _silu_case(count, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    pre = (torch.randn(count, device=dev, generator=g) * 4).to(bf)
    pre[:8] = torch.tensor([-1e4, -200., -90., -30., 30., 90., 200., 1e4], device=dev).to(bf)   # saturated SiLU
    dout = torch.randn(count, device=dev, generator=g).to(bf)
    buf = torch.full((count + 64,), float("nan"), device=dev, dtype=bf)
    got = ops.silu_bwd(pre, dout, buf[:count])
    assert_nan(buf[count:], "past count")
    return pre, dout, got


def _silu_bound(ref, pre, dout):
    # bf16 rounding of the result + fp32 intermediates (__expf: a few ulp) relative to |dy| (1 + |x|)
    return U_BF16 * ref.abs() + 2.0 ** -18 * dout.double().abs() * (1 + pre.double().abs())


@pytest.mark.parametrize("count", [2, 1000, 3 * 2 ** 16 + 6])
def test_silu_bwd(count):
    pre, dout, got = _silu_case(max(count, 8), seed=count)
    ref = _silu_grad64(pre.double(), dout.double())
    assert_close(got, ref, _silu_bound(ref, pre, dout), 2.0 ** -8, f"count={count}")
    assert float(got[0]) == 0.0 and float(got[7]) == float(dout[7]), "saturated SiLU: 0 and the identity"


def test_silu_bwd_in_place_and_sensitivity():
    from naturalspeech2_pytorch_b200 import ops
    pre, dout, got = _silu_case(4096, seed=9)
    ref = _silu_grad64(pre.double(), dout.double())
    inplace = pre.clone()
    ops.silu_bwd(inplace, dout)
    assert torch.equal(inplace, got), "dpre aliasing pre gives the same result"
    wrong = dout.double() * torch.sigmoid(pre.double())          # the x (1 - s) term dropped
    assert_rejects(got, wrong, _silu_bound(ref, pre, dout), 2.0 ** -8, "sigmoid-only derivative")


# ---------------------------------------------------------------------------------------------------------------
# embedding_bwd
# ---------------------------------------------------------------------------------------------------------------
def _emb_case(rows_table, dim, B, T, seed, start_zero=True):
    from naturalspeech2_pytorch_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    pad = rows_table - 1
    ids = torch.randint(0, rows_table // 2, (B, T), device=dev, generator=g)   # upper half of the table never occurs
    ids[:, :3] = 1                                                              # one id repeated in every sample
    ids[-1, T - 5:] = -1                                                        # padding -> the pad row
    de = torch.randn(B, T, dim, device=dev, generator=g)
    buf = torch.full(((rows_table + 3) * dim,), float("nan"), device=dev)
    table = buf[:rows_table * dim].view(rows_table, dim)
    table.copy_(torch.zeros(rows_table, dim, device=dev) if start_zero else torch.randn(rows_table, dim, device=dev, generator=g))
    start = table.clone()
    ops.embedding_bwd(ids, de, table, pad)
    assert_nan(buf[rows_table * dim:], "past the table")
    return ids, de, start, table, pad


def _emb_ref(ids, de, rows_table, pad):
    idx = ids.masked_fill(ids < 0, pad).flatten()
    d = de.double().reshape(-1, de.shape[-1])
    ref = torch.zeros(rows_table, de.shape[-1], dtype=torch.float64, device=dev).index_add_(0, idx, d)
    mag = torch.zeros_like(ref).index_add_(0, idx, d.abs())
    return ref, mag


@pytest.mark.parametrize("dim", [64, 200])
def test_embedding_bwd_repeats_pad_and_unused_rows(dim):
    rows_table = 41
    ids, de, start, got, pad = _emb_case(rows_table, dim, 3, 37, seed=dim)
    ref, mag = _emb_ref(ids, de, rows_table, pad)
    assert_close(got, ref, acc_eps(ids.numel()) * mag + U_F32 * ref.abs(), acc_eps(ids.numel()) * 4, f"dim={dim}")
    occurs = torch.zeros(rows_table, dtype=torch.bool, device=dev)
    occurs[ids.masked_fill(ids < 0, pad).flatten()] = True
    assert bool(occurs[pad]) and torch.count_nonzero(got[pad]) == dim, "the pad row receives gradient"
    assert torch.count_nonzero(got[~occurs]) == 0, "rows that never occur stay exactly zero"


def test_embedding_bwd_accumulates_and_sensitivity():
    rows_table, dim = 41, 128
    ids, de, start, got, pad = _emb_case(rows_table, dim, 2, 50, seed=3, start_zero=False)
    ref, mag = _emb_ref(ids, de, rows_table, pad)
    bound = acc_eps(ids.numel()) * mag + U_F32 * (got.double().abs() + start.double().abs())
    assert_close(got.double() - start.double(), ref, bound, acc_eps(ids.numel()) * 4, "accumulate")
    wrong, _ = _emb_ref(torch.where(ids >= 0, (ids + 1) % (rows_table - 1), ids), de, rows_table, pad)
    assert_rejects(got.double() - start.double(), wrong, bound, acc_eps(ids.numel()) * 4, "ids off by one")


# ---------------------------------------------------------------------------------------------------------------
# expand_encodings_bwd
# ---------------------------------------------------------------------------------------------------------------
def _expand_case(B, T, D, L, table_rows, seed, stride_pad=24):
    """dcond as a column window of a wider NaN-padded buffer; durations with zeros and short samples (idx = -1
    tails); coarse bins drawn from a few values so samples share table rows."""
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200.encoders import frames_to_text_index
    g = torch.Generator(device=dev).manual_seed(seed)
    dur = torch.randint(0, 2 * L // T + 1, (B, T), device=dev, generator=g)
    dur[:, 1] = 0
    dur[0, -2:] = 0
    dur = torch.minimum(dur, torch.full_like(dur, L))
    while bool((dur.sum(-1) > L).any()):                       # fit every sample into L frames
        dur = torch.where((dur.sum(-1, keepdim=True) > L) & (dur > 0), dur - 1, dur)
    idx = frames_to_text_index(dur, length=L)
    coarse = torch.randint(1, 6, (B, T), device=dev, generator=g).int() * (table_rows // 6)
    wide = torch.full((B, L, D + stride_pad), float("nan"), device=dev)
    wide[..., :D] = torch.randn(B, L, D, device=dev, generator=g)
    dcond = wide[..., :D]
    dphon = torch.zeros(B, T, D, device=dev)
    tbuf = torch.full(((table_rows + 2) * D,), float("nan"), device=dev)
    dtable = tbuf[:table_rows * D].view(table_rows, D)
    dtable.zero_()
    ops.expand_encodings_bwd(dcond, coarse, idx, dphon, dtable)
    assert_nan(tbuf[table_rows * D:], "past the table")
    return dur, idx, coarse, dcond, dphon, dtable


def _expand_ref(idx, coarse, dcond, T, table_rows):
    B, L, D = dcond.shape
    onehot = torch.zeros(B, L, T, dtype=torch.float64, device=dev)
    valid = idx >= 0
    onehot[valid.nonzero(as_tuple=True) + (idx[valid].long(),)] = 1.0
    dphon = torch.einsum("bnt,bnd->btd", onehot, dcond.double())
    mag = torch.einsum("bnt,bnd->btd", onehot, dcond.double().abs())
    dtab = torch.zeros(table_rows, D, dtype=torch.float64, device=dev).index_add_(0, coarse.long().flatten(),
                                                                                   dphon.reshape(-1, D))
    tmag = torch.zeros_like(dtab).index_add_(0, coarse.long().flatten(), mag.reshape(-1, D))
    return dphon, mag, dtab, tmag


@pytest.mark.parametrize("B,T,D,L", [
    (2, 7, 128, 64),      # two whole 32-frame blocks, one 128-channel block
    (3, 21, 200, 203),    # L and D not multiples of any tile; runs cut by block boundaries
    (1, 5, 512, 1030),    # long phonemes spanning many blocks
])
def test_expand_encodings_bwd(B, T, D, L):
    dur, idx, coarse, dcond, dphon, dtable = _expand_case(B, T, D, L, 48, seed=B * 1000 + L)
    ref, mag, tref, tmag = _expand_ref(idx, coarse, dcond, T, 48)
    assert_close(dphon, ref, acc_eps(L) * mag + U_F32 * ref.abs(), acc_eps(L) * 4, "dphon")
    assert_close(dtable, tref, acc_eps(B * L) * tmag + U_F32 * tref.abs(), acc_eps(B * L) * 4, "dtable")
    assert torch.count_nonzero(dphon[dur == 0]) == 0, "zero-duration phonemes get exact zeros"
    used = torch.zeros(48, dtype=torch.bool, device=dev)
    used[coarse[dur > 0].long()] = True
    assert torch.count_nonzero(dtable[~used]) == 0, "table rows no frame maps to stay exactly zero"


def test_expand_encodings_bwd_sensitivity():
    dur, idx, coarse, dcond, dphon, dtable = _expand_case(2, 9, 128, 150, 48, seed=4)
    ref, mag, _, _ = _expand_ref(idx, coarse, dcond, 9, 48)
    late = torch.cat((torch.full_like(idx[:, :1], -1), idx[:, :-1]), dim=1)   # every frame attributed one frame late
    wrong, _, _, _ = _expand_ref(late, coarse, dcond, 9, 48)
    assert_rejects(dphon, wrong, acc_eps(150) * mag + U_F32 * ref.abs(), acc_eps(150) * 4, "alignment one frame late")
