"""CPU: the host-side argument checks of the RVQ decode and cross-entropy wrappers and of ns2_rvq_ce's C ABI (each
rejection happens before any launch), and the empty-codes decode."""
import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_rvq_ce_c_abi_rejects_bad_arguments_before_launch(lib):
    """Dummy non-NULL device pointers are never dereferenced: every call fails its argument check."""
    before = lib.ns2_launch_count()
    p = 16
    assert lib.ns2_rvq_ce(p, 4, 128, p, p, 1, 256, p, None, p, p, None) < 0      # NULL target codes
    assert b"NULL" in lib.ns2_last_error()
    assert lib.ns2_rvq_ce(p, 4, 128, p, p, 1, 256, p, p, p, None, None) < 0      # NULL loss
    assert lib.ns2_rvq_ce(p, 4, 64, p, p, 1, 256, p, p, p, p, None) < 0         # d != 128
    assert lib.ns2_rvq_ce(p, 4, 128, p, p, 1, 31, p, p, p, p, None) < 0         # k < 32
    assert lib.ns2_rvq_ce(p, 4, 128, p, p, 0, 256, p, p, p, p, None) < 0        # q = 0
    assert lib.ns2_rvq_ce(p, 4, 128, p, p, -1, 256, p, p, p, p, None) < 0       # q < 0
    assert lib.ns2_rvq_ce(p, 0, 128, p, p, 1, 256, p, p, p, p, None) < 0        # no frames
    assert lib.ns2_rvq_ce(p, -3, 128, p, p, 1, 256, p, p, p, p, None) < 0       # negative frames
    assert lib.ns2_launch_count() == before


def _codes(F, Q, dtype=torch.int64):
    return torch.zeros(F, Q, dtype=dtype)


@pytest.mark.parametrize("case, match", [
    ("int32 codes", "codes must be torch.int64"),
    ("codes last dim != Q", r"codes must have shape \(\*, 8\)"),
    ("1-d codes", r"codes must have shape"),
    ("strided codes", "codes must be contiguous"),
    ("fp16 codebooks", "codebooks must be torch.float32"),
    ("codebooks d != 128", r"codebooks must have shape \(\*, \*, 128\)"),
    ("fp64 out", "out must be torch.float32"),
    ("out wrong rows", r"out must have shape \(4, 128\)"),
    ("strided out", "out must be contiguous"),
    ("CPU codes", "codes must be a CUDA tensor"),
])
def test_rvq_decode_rejects_bad_arguments_before_launch(lib, case, match):
    from naturalspeech2_pytorch_b200 import ops
    cb = torch.zeros(8, 128, 128)
    args = {
        "int32 codes": (_codes(4, 8, torch.int32), cb, None),
        "codes last dim != Q": (_codes(8, 4), cb, None),
        "1-d codes": (torch.zeros(32, dtype=torch.int64), cb, None),
        "strided codes": (_codes(8, 4).t(), cb, None),
        "fp16 codebooks": (_codes(4, 8), cb.half(), None),
        "codebooks d != 128": (_codes(4, 8), torch.zeros(8, 128, 64), None),
        "fp64 out": (_codes(4, 8), cb, torch.zeros(4, 128, dtype=torch.float64)),
        "out wrong rows": (_codes(4, 8), cb, torch.zeros(5, 128)),
        "strided out": (_codes(4, 8), cb, torch.zeros(128, 4).t()),
        "CPU codes": (_codes(4, 8), cb, torch.zeros(4, 128)),
    }[case]
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match=match):
        ops.rvq_decode(*args[:2], out=args[2])
    assert lib.ns2_launch_count() == before


@pytest.mark.parametrize("case, match", [
    ("fp64 codebooks", "codebooks must be torch.float32"),
    ("codebooks d != 128", r"codebooks must have shape \(\*, \*, 128\)"),
    ("frames d != 128", r"frames must have shape \(\*, 128\)"),
    ("fp64 cn2", "cn2 must be torch.float32"),
    ("cn2 of another K", r"cn2 must have shape \(2, 64\)"),
    ("flat cn2", r"cn2 must have shape \(2, 64\)"),
    ("strided cn2", "cn2 must be contiguous"),
    ("int32 own codes", "own_codes must be torch.int64"),
    ("target codes of another F", r"target_codes must have shape \(6, 2\)"),
    ("CPU tensors", "frames must be a CUDA tensor"),
])
@pytest.mark.parametrize("op", ["rvq_ce", "rvq_ce_bwd"])
def test_rvq_ce_wrappers_reject_bad_arguments_before_launch(lib, op, case, match):
    from naturalspeech2_pytorch_b200 import ops
    F, Q, K = 6, 2, 64
    a = dict(frames=torch.zeros(F, 128), codebooks=torch.zeros(Q, K, 128), cn2=torch.zeros(Q, K),
             own_codes=_codes(F, Q), target_codes=_codes(F, Q))
    bad = {
        "fp64 codebooks": dict(codebooks=a["codebooks"].double()),
        "codebooks d != 128": dict(codebooks=torch.zeros(Q, K, 64)),
        "frames d != 128": dict(frames=torch.zeros(F, 64)),
        "fp64 cn2": dict(cn2=a["cn2"].double()),
        "cn2 of another K": dict(cn2=torch.zeros(Q, 2 * K)),
        "flat cn2": dict(cn2=torch.zeros(Q * K)),
        "strided cn2": dict(cn2=torch.zeros(K, Q).t()),
        "int32 own codes": dict(own_codes=_codes(F, Q, torch.int32)),
        "target codes of another F": dict(target_codes=_codes(F + 1, Q)),
        "CPU tensors": {},
    }[case]
    a.update(bad)
    extra = (torch.ones(1),) if op == "rvq_ce_bwd" else ()
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match=match):
        getattr(ops, op)(a["frames"], a["codebooks"], a["cn2"], a["own_codes"], a["target_codes"], *extra)
    assert lib.ns2_launch_count() == before


def test_get_emb_from_indices_empty_and_shape_checks():
    """Empty codes decode to correctly shaped empties without a launch, as `quantize` does for empty frames; codes whose
    last dimension is not Q, and float codes, are rejected."""
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    codec = EncodecRVQ(torch.randn(8, 1024, 128))
    for shape in ((0, 8), (2, 0, 8), (0, 3, 8)):
        for dtype in (torch.int64, torch.int32):
            emb = codec.get_emb_from_indices(torch.empty(shape, dtype=dtype))
            assert emb.shape == shape[:-1] + (128,) and emb.dtype == torch.float32 and emb.device.type == "cpu"
    with pytest.raises(ValueError, match=r"\(\.\.\., 8\)"):
        codec.get_emb_from_indices(torch.zeros(3, 4, dtype=torch.int64))
    with pytest.raises(ValueError, match="integer"):
        codec.get_emb_from_indices(torch.zeros(3, 8))
