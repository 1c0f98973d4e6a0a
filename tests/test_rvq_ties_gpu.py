"""GPU: RVQ encode (`ops.rvq_prepare` / `ops.rvq_encode` through `EncodecRVQ`) on exact and near ties, bit-exact against
the fp64 argmin oracle (lowest index wins on ties).

The kernel filters with an fp16 tensor-core score and re-scores in fp64 every code whose approximate score lies in
the error band of the best one.  Inside each 128-code chunk the prepared codebook is permuted so that a thread scans
one 32-code block; column half 0 (codes 0-63 of a chunk) and half 1 (64-127) keep separate top-8 lists; a row whose
band holds two codes of one 32-code block rescans that block ("crowded", stats[3]); a list that is entirely inside the
band forces an exact scan of the whole codebook (stats[2]).  The ties below are built from small integers and powers
of two, so every distance is exact in fp32 and fp64 and the oracle's tie really is a tie.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
TIE_DIMS = (100, 101, 102)   # directions of the tie offsets v (codeword = m + v)
U_CODE = 64                  # stage-0 code that brings a frame onto m for a stage-1 tie


def _e(d, scale=1.0):
    v = np.zeros(128, np.float32)
    v[d] = scale
    return v


def _codebooks(Q, K, seed):
    return np.random.default_rng(seed).standard_normal((Q, K, 128)).astype(np.float32)


def _place(cb, q, codes, base_dim, sign=1.0):
    """Codes equidistant (distance 1) from m = 8 e_base: a pair m + s v, m - s v, or three codes m + v_i with
    orthogonal v_i.  Returns m."""
    m = _e(base_dim, 8.0)
    if len(codes) == 2:
        cb[q, codes[0]] = m + sign * _e(TIE_DIMS[0])
        cb[q, codes[1]] = m - sign * _e(TIE_DIMS[0])
    else:
        for c, d in zip(codes, TIE_DIMS):
            cb[q, c] = m + _e(d)
    return m


def _frame_for_stage(cb, m, stage, base_dim):
    """A frame whose residual at `stage` is exactly m: m itself at stage 0; at stage 1 stage-0 code U_CODE is set to
    u = 16 e_(base+1) and the frame is m + u, so the stage-0 winner is u and the residual m + u - u = m."""
    if stage == 0:
        return m.copy()
    u = _e(base_dim + 1, 16.0)
    cb[0, U_CODE] = u
    return m + u


def _encode(frames, cb):
    from naturalspeech2_pytorch_b200 import EncodecRVQ, _lib
    stats = torch.zeros(_lib.NS2_RVQ_STATS_LEN, dtype=torch.int64, device=dev)
    codes, _ = EncodecRVQ(torch.from_numpy(cb)).cuda().quantize(torch.from_numpy(frames).cuda(), stats=stats)
    return codes.cpu().numpy(), stats[:4].cpu().tolist()


def _oracle(frames, cb):
    from oracle import rvq_oracle
    return rvq_oracle.encode(frames, cb, return_gaps=True)


def _tie_case(K, codes, stage, sign, F=6, tie_rows=(1, 4), seed=0):
    Q = 2
    cb = _codebooks(Q, K, seed)
    m = _place(cb, stage, codes, 10, sign)
    tie_frame = _frame_for_stage(cb, m, stage, 10)
    frames = np.random.default_rng(seed + 1).standard_normal((F, 128)).astype(np.float32)
    for r in tie_rows:
        frames[r] = tie_frame
    got, stats = _encode(frames, cb)
    ref, gaps = _oracle(frames, cb)
    # the construction is a real tie, resolved to the lowest index by the oracle
    for r in tie_rows:
        assert gaps[r, stage] == 0.0 and ref[r, stage] == min(codes), (r, ref[r], gaps[r])
    np.testing.assert_array_equal(got, ref)
    assert stats[1] > 0, "the tie rows must take the exact re-score"
    return got, ref


PLACEMENTS = [
    (256, (3, 17)),          # same 32-code block (block 0)
    (256, (40, 100)),        # the two column halves of chunk 0
    (256, (10, 200)),        # chunks 0 / 1, the lower index in list a (half 0) is seen first
    (256, (70, 130)),        # chunks 0 / 1, the higher index is in list a (half 0 of chunk 1) and is seen first
    (256, (20, 50, 200)),    # three-way tie across blocks 0, 1 and 6
    (128, (0, 127)),         # K = 128: a single chunk, first and last code
    (128, (126, 127)),       # K = 128: the last two codes of the only chunk
    (2048, (2046, 2047)),    # K = MAX_K: the top of the 11-bit index field of the packed keys
    (2048, (5, 2047)),       # K = MAX_K: first and last chunk
]


@pytest.mark.parametrize("sign", [1.0, -1.0], ids=["a=m+v", "a=m-v"])
@pytest.mark.parametrize("stage", [
    0,   # the residual is the raw frame
    1,   # the residual is frame - stage-0 codeword
])
@pytest.mark.parametrize("K,codes", PLACEMENTS)
def test_rvq_equal_distance_ties(K, codes, stage, sign):
    _tie_case(K, codes, stage, sign, seed=K + stage)


@pytest.mark.parametrize("F,tie_rows", [
    (1, (0,)),             # a single frame
    (127, (125, 126)),     # the last rows of a partial CTA
    (128, (126, 127)),     # the last rows of a full CTA
    (129, (127, 128)),     # one tie row in each CTA; the second CTA holds only that row
])
def test_rvq_ties_in_last_cta(F, tie_rows):
    _tie_case(256, (40, 100), 0, 1.0, F=F, tie_rows=tie_rows, seed=F)


def test_rvq_tie_sensitivity_swapped_codes():
    """A reference with the two codes of a tie swapped is rejected (the comparison is bit-exact)."""
    got, ref = _tie_case(256, (10, 200), 0, 1.0, seed=5)
    wrong = ref.copy()
    wrong[[1, 4], 0] = 200
    assert (got != wrong).any()


@pytest.mark.parametrize("winner_first", [True, False], ids=["winner-lower-index", "winner-higher-index"])
def test_rvq_near_ties(winner_first):
    """Distances 16 and 16 + 2^-18 from m = 8 e_10: the scores -48 and -48 + 2^-18 differ by one fp32 ulp, far inside
    the fp16 filter's error band, so only the fp64 re-score separates them."""
    K, Q = 256, 2
    cb = _codebooks(Q, K, 31)
    m = _e(10, 8.0)
    near, far = (20, 150) if winner_first else (150, 20)
    cb[0, near] = m + _e(TIE_DIMS[0], 4.0)
    cb[0, far] = m + _e(TIE_DIMS[0], 4.0) + _e(TIE_DIMS[1], 2.0 ** -9)
    frames = np.random.default_rng(32).standard_normal((10, 128)).astype(np.float32)
    frames[[2, 9]] = m
    got, stats = _encode(frames, cb)
    ref, gaps = _oracle(frames, cb)
    assert (ref[[2, 9], 0] == near).all() and (gaps[[2, 9], 0] > 0).all()
    np.testing.assert_array_equal(got, ref)
    assert stats[1] > 0


def test_rvq_degenerate_codebook_full_scan():
    """All codewords equal: every code is in the band, the top-8 lists overflow and the whole codebook is scanned."""
    K, Q = 256, 2
    cb = np.broadcast_to(_codebooks(Q, 1, 41), (Q, K, 128)).copy()
    frames = np.random.default_rng(42).standard_normal((200, 128)).astype(np.float32)
    got, stats = _encode(frames, cb)
    ref, _ = _oracle(frames, cb)
    assert (ref == 0).all()
    np.testing.assert_array_equal(got, ref)
    assert stats[2] > 0, stats


def test_rvq_crowded_block():
    """Three equidistant codes, two of them (5, 6) in one 32-code block: that block is rescanned exactly."""
    K, Q = 256, 2
    cb = _codebooks(Q, K, 51)
    m = _e(10, 8.0)
    cb[0, 5] = m + _e(TIE_DIMS[0])
    cb[0, 6] = m - _e(TIE_DIMS[0])
    cb[0, 200] = m + _e(TIE_DIMS[1])
    frames = np.random.default_rng(52).standard_normal((40, 128)).astype(np.float32)
    frames[[0, 17, 39]] = m
    got, stats = _encode(frames, cb)
    ref, _ = _oracle(frames, cb)
    assert (ref[[0, 17, 39], 0] == 5).all()
    np.testing.assert_array_equal(got, ref)
    assert stats[3] > 0, stats


@pytest.mark.parametrize("K", [
    4096,   # larger than MAX_K = 2048 (the 11-bit index field of the packed keys)
    192,    # not a multiple of the 128-code chunk
])
def test_rvq_rejects_unsupported_codebook_size(K):
    from naturalspeech2_pytorch_b200 import _lib, ops
    cb = torch.zeros(1, K, 128, device=dev)
    frames = torch.zeros(4, 128, device=dev)
    dummy = (torch.zeros(8, device=dev, dtype=torch.float16), torch.zeros(K, device=dev), torch.zeros(2, device=dev))
    before = ops.launch_count()
    with pytest.raises(_lib.Ns2Error, match="codebook size"):
        ops.rvq_encode(frames, cb, dummy)
    if K % 128:
        with pytest.raises(_lib.Ns2Error, match="codebook size"):
            ops.rvq_prepare(cb)
    assert ops.launch_count() == before, "a rejected call must not launch a kernel"
