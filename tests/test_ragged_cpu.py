"""CPU: the C entry points behind per-sample lengths reject NULL and invalid arguments before any launch, and the
Python side rejects bad lengths and unsupported combinations before any CUDA call."""
import ctypes

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_arguments(lib):
    from naturalspeech2_pytorch_b200._lib import AttnArgs
    before = lib.ns2_launch_count()
    a = AttnArgs(kv_lens=16)
    assert lib.ns2_attn_fwd(ctypes.byref(a), None) < 0                     # NULL q / k / v / out
    assert lib.ns2_attn_fwd(None, None) < 0
    assert lib.ns2_groupnorm_silu(16, 2, 8, 100, 8, 16, 16, 1e-5, None, 16, None, 16, None) < 0   # 100 % 8
    assert lib.ns2_mean_rows(None, 2, 8, 64, 16, 16, None) < 0
    assert lib.ns2_cond_inject(16, 16, 16, None, 2, 8, 8, 64, 16, 16, None) < 0   # drop mask without null_cond
    assert lib.ns2_mask_rows(16, 1, 64, 512, 2, 8, 64, None, None) < 0
    assert lib.ns2_mask_rows(16, 1, 32, 512, 2, 8, 64, 16, None) < 0                    # row stride < cols
    assert lib.ns2_mask_rows(None, 1, 64, 512, 0, 8, 64, None, None) == 0               # empty: nothing to do
    args = (16, 64, 640, 10, 16, 16, 64, 640, 10, 16, 2, 64, 16, 64, 1280)
    assert lib.ns2_pack_rows(*args, 19, None) < 0                                        # out_rows < 10 + 10
    assert lib.ns2_pack_rows(*args[:4], None, *args[5:], 20, None) < 0                   # NULL a_lens
    bad_cols = args[:11] + (62,) + args[12:]
    assert lib.ns2_pack_rows(*bad_cols, 20, None) < 0
    assert b"multiples of 4" in lib.ns2_last_error()
    assert lib.ns2_launch_count() == before


def test_attention_rejects_kv_lens_with_dropout(lib):
    """Key padding has no dropout kernel: ns2_attn_fwd refuses kv_lens with a dropout of p > 0 before it launches."""
    from naturalspeech2_pytorch_b200._lib import AttnArgs, Dropout
    before = lib.ns2_launch_count()
    d = Dropout(1, 0, 0.5)
    assert lib.ns2_attn_fwd(ctypes.byref(AttnArgs(kv_lens=16, dropout=ctypes.pointer(d))), None) < 0
    assert b"kv_lens" in lib.ns2_last_error()
    assert lib.ns2_launch_count() == before


def test_lengths_rejected_on_the_host():
    """ops.lengths checks the values it is given before it creates any CUDA tensor."""
    from naturalspeech2_pytorch_b200 import ops
    for lens, n in (([0, 3], 5), ([1, 6], 5), ([1, 2, 3], 5), ([1], 5)):
        with pytest.raises(ValueError):
            ops.lengths(lens, 2, n, device="cuda")
    with pytest.raises(ValueError):
        ops.lengths(torch.tensor([1.0, 2.0]), 2, 5, device="cuda")
    with pytest.raises(ValueError):
        ops.lengths(torch.tensor([[1, 2]]), 2, 5, device="cuda")
    with pytest.raises(ValueError):
        ops.lengths([-1, 0], 2, None, device="cuda", lo=0)
    with pytest.raises(ValueError):   # a CPU tensor where the kernels need device lengths
        ops.mask_rows(torch.zeros(2, 3, 4), torch.tensor([1, 2], dtype=torch.int32))


def test_python_rejections_before_cuda():
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=10)
    with pytest.raises(NotImplementedError):
        cn(prompt=torch.zeros(1, 4, 128), text=torch.zeros(1, 3, dtype=torch.long), mode="train", phoneme_lens=[3])
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True)
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=2, conditioner=cn)
    with pytest.raises(ValueError, match="encoded latents"):
        ns.sample(length=8, prompt=torch.zeros(1, 4800), text=torch.zeros(1, 3, dtype=torch.long), prompt_lens=[1])
    with pytest.raises(ValueError, match="cond_lens"):
        ns.sample(length=8, prompt=torch.zeros(1, 4, 128), text=torch.zeros(1, 3, dtype=torch.long), cond_lens=[1])
    with pytest.raises(ValueError):
        model(torch.zeros(1, 8, 128), torch.zeros(1), _conditioning={}, prompt_lens=[1])
    uncond = NaturalSpeech2(Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1),
                            target_sample_hz=24000, timesteps=2)
    with pytest.raises(ValueError):
        uncond.sample(length=8, prompt_lens=[1])
