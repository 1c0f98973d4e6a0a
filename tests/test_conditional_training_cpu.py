"""CPU: host-side pieces of conditional training — the average_over_durations restatement against the reference's
values (tests/golden/grads_cond_train.npz), Conditioner(mode="train") argument checks, NaturalSpeech2.forward's
`duration` hand-off, and the data-parallel all-reduce of encoder gradients (gloo, world_size 2)."""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN


def test_average_over_durations_matches_reference_bit_for_bit():
    from naturalspeech2_pytorch_b200.encoders import average_over_durations
    z = np.load(GOLDEN / "grads_cond_train.npz")
    vals, durs = torch.from_numpy(z["avg_values"]), torch.from_numpy(z["avg_durs"])
    np.testing.assert_array_equal(average_over_durations(vals, durs).numpy(), z["avg_out"])
    np.testing.assert_array_equal(average_over_durations(vals[:, :1], durs.float()).numpy(), z["avg_out_float_durs"])
    from golden.make_golden_cond_train import cond_train_inputs
    from naturalspeech2_pytorch_b200.encoders import f0_to_coarse
    for case in ("e2e_small", "e2e_wide"):   # the per-phoneme pitch of the end-to-end goldens -> their coarse bins
        inp = cond_train_inputs(case)
        np.testing.assert_array_equal(inp["duration"].numpy(), z[f"{case}::in_duration"])
        avg = average_over_durations(inp["pitch"], inp["duration"])
        np.testing.assert_array_equal(f0_to_coarse(avg[:, 0]).numpy(), z[f"{case}::coarse"])


@pytest.fixture(scope="module")
def conditioner():
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    return Conditioner(dim_codebook=128, num_phoneme_tokens=20)


def test_conditioner_train_mode_argument_errors(conditioner):
    prompt, text = torch.zeros(2, 10, 128), torch.zeros(2, 5, dtype=torch.long)
    pitch = torch.zeros(2, 30)
    ok = torch.tensor([[3, 4, 5, 6, 7], [1, 1, 1, 1, 1]])
    with pytest.raises(NotImplementedError, match="duration"):
        conditioner(prompt=prompt, text=text, pitch=pitch, mode="train")
    with pytest.raises(ValueError, match="pitch"):
        conditioner(prompt=prompt, text=text, duration=ok, mode="train")
    with pytest.raises(ValueError, match="non-negative"):
        conditioner(prompt=prompt, text=text, pitch=pitch, duration=ok - 2, mode="train")
    with pytest.raises(ValueError, match="past the 30 frames"):
        conditioner(prompt=prompt, text=text, pitch=pitch, duration=ok * 2, mode="train")
    with pytest.raises(ValueError, match=r"\(B, T\)"):
        conditioner(prompt=prompt, text=text, pitch=pitch, duration=ok[:, :4], mode="train")
    with pytest.raises(ValueError, match="whole frame counts"):
        conditioner(prompt=prompt, text=text, pitch=pitch, duration=ok + 0.5, mode="train")
    with pytest.raises(NotImplementedError):
        conditioner(prompt=prompt, text=text, mode="align")


def test_conditioner_grad_reducer_reaches_both_encoders(conditioner):
    from naturalspeech2_pytorch_b200.parallel import GradReducer
    red = GradReducer()
    conditioner.grad_reducer = red
    assert conditioner.prompt_enc.grad_reducer is red and conditioner.phoneme_enc.grad_reducer is red
    conditioner.grad_reducer = None
    assert conditioner.prompt_enc.grad_reducer is None and conditioner.phoneme_enc.grad_reducer is None


def test_naturalspeech2_forward_passes_duration_only_when_given():
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    seen = []

    class Stop(Exception):
        pass

    def conditioner(**kw):
        seen.append(kw)
        raise Stop

    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=128, condition_on_prompt=True)
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=2, conditioner=conditioner)
    lat, prompt, text, pitch = torch.zeros(1, 16, 128), torch.zeros(1, 8, 128), torch.zeros(1, 4, dtype=torch.long), torch.zeros(1, 16)
    with pytest.raises(Stop):
        ns(lat, text=text, prompt=prompt, pitch=pitch)
    assert "duration" not in seen[-1] and seen[-1]["mode"] == "train"
    dur = torch.full((1, 4), 4)
    with pytest.raises(Stop):
        ns(lat, text=text, prompt=prompt, pitch=pitch, duration=dur)
    assert seen[-1]["duration"] is dur


def _encoder_reducer_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from naturalspeech2_pytorch_b200 import encoders, parallel
    parallel.init_from_env(backend="gloo")
    enc = encoders.PhonemeEncoder(num_tokens=10, dim=64, dim_hidden=128, depth=1, heads=2)
    red = parallel.GradReducer(coalesce_below=4096)
    # the encoder's kernels need a GPU: stand-ins with the same contract give rank-dependent gradients, so the test
    # checks what the autograd node does with them (hand every buffer to the reducer, finish, return the averages)
    enc._train_forward = lambda x: (x.float().unsqueeze(-1).expand(*x.shape, 128).clone(), None)
    enc._train_backward = lambda saved, d: {n: torch.full(p.shape, float(rank + 1)) * (i + 1)
                                            for i, (n, p) in enumerate(enc.named_parameters())}
    out = encoders._EncoderFunction.apply(enc, red, torch.zeros(2, 3, dtype=torch.long), *enc.parameters())
    out.sum().backward()
    ok = all(torch.allclose(p.grad, torch.full(p.shape, 1.5 * (i + 1))) for i, (_, p) in enumerate(enc.named_parameters()))
    q.put((rank, ok, red.bytes_reduced))
    dist.destroy_process_group()


def test_encoder_gradients_are_averaged_over_ranks_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_encoder_reducer_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, ok, nbytes in res:
        assert ok and nbytes > 0
