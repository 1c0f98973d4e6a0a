"""CPU: host-side argument checks of the duration / pitch predictor's backward entry points, the predictor's autograd
node with stand-in kernels (several inputs and outputs, a trunk without gradient, GradReducer over a 2-rank gloo
group), and the loss weights' plumbing."""
import os

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_backward_entry_points_reject_bad_arguments_before_any_launch(lib):
    before = lib.ns2_launch_count()
    p = 1 << 12                                            # dummy aligned address, never dereferenced
    gn = lambda batch, rows, ch, groups, *ptrs: lib.ns2_groupnorm_silu_bwd(  # noqa: E731
        p, batch, rows, ch, groups, p, p, 1e-5, p, p, p, *ptrs, None)
    assert gn(2, 8, 48, 8, p, p) < 0 and b"multiple of 4" in lib.ns2_last_error()          # 6 channels per group
    assert gn(2, 8, 100, 8, p, p) < 0 and b"bad sizes" in lib.ns2_last_error()             # 100 % 8 != 0
    assert gn(2, 8, 2048 * 2, 2, p, p) < 0 and b"1024" in lib.ns2_last_error()             # cpg 2048
    assert gn(65536, 8, 512, 8, p, p) < 0 and b"65535" in lib.ns2_last_error()
    assert gn(2, 8, 512, 8, None, p) < 0 and b"null" in lib.ns2_last_error()
    assert lib.ns2_groupnorm_silu_bwd(p + 4, 2, 8, 512, 8, p, p, 1e-5, p, p, p, p, p, None) < 0
    assert b"aligned" in lib.ns2_last_error()
    assert lib.ns2_groupnorm_silu_bwd(None, 2, 8, 512, 8, p, p, 1e-5, p, p, p, p, p, None) < 0
    rd = lambda rows, dim, x=p, dw=p: lib.ns2_rowdot_bwd(x, rows, dim, p, p, p, p, p, dw, p, None)  # noqa: E731
    assert rd(4, 10) < 0 and b"bad sizes" in lib.ns2_last_error()                          # dim % 4 != 0
    assert rd(-1, 16) < 0
    assert rd(4, 16, dw=None) < 0 and b"null" in lib.ns2_last_error()
    assert rd(4, 16, x=None) < 0 and b"null" in lib.ns2_last_error()
    assert rd(4, 16, x=p + 4) < 0 and b"aligned" in lib.ns2_last_error()
    assert lib.ns2_launch_count() == before


def test_header_constant_matches_the_binding():
    import re
    from pathlib import Path
    from naturalspeech2_pytorch_b200 import _lib
    h = (Path(__file__).resolve().parent.parent / "include" / "ns2_b200.h").read_text()
    assert int(re.search(r"#define NS2_ROWDOT_BWD_ROWS (\d+)", h).group(1)) == _lib.NS2_ROWDOT_BWD_ROWS


def test_loss_weights_are_read_not_swallowed():
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512, condition_on_prompt=True)
    ns = NaturalSpeech2(model, target_sample_hz=24000, duration_loss_weight=0.5, pitch_loss_weight=2.0, foo=1)
    assert (ns.duration_loss_weight, ns.pitch_loss_weight) == (0.5, 2.0) and ns.conditioning_kwargs == {"foo": 1}
    assert (NaturalSpeech2(model, target_sample_hz=24000).duration_loss_weight, ns.pitch_loss_weight) == (1.0, 2.0)
    assert Conditioner.train_duration_pitch is False


def _stand_ins(pred, rank):
    """The predictor's kernels need a GPU: stand-ins with its contract (two inputs, two outputs, input gradients under
    _INPUT_GRADS, None for the parameters of a trunk without upstream gradient)."""
    from naturalspeech2_pytorch_b200 import encoders
    pred._train_forward = lambda x, pr: ((x.sum(-1) * 2, x.sum(-1) + pr.sum((1, 2))[:, None]), None)

    def backward(saved, d_dur, d_pitch):
        grads = {}
        for i, (n, p) in enumerate(pred.named_parameters()):
            skip = (n.startswith("to_pitch_pred.") and d_pitch is None) or (n.startswith("to_duration_pred.") and d_dur is None)
            grads[n] = None if skip else torch.full(p.shape, float(rank + 1)) * (i + 1)
        grads[encoders._INPUT_GRADS] = (torch.full((2, 3, 128), 3.0), torch.full((2, 5, 128), 4.0))
        return grads
    pred._train_backward = backward


def _predictor_reducer_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from naturalspeech2_pytorch_b200 import encoders, parallel
    parallel.init_from_env(backend="gloo")
    cond = encoders.Conditioner.__new__(encoders.Conditioner)
    torch.nn.Module.__init__(cond)
    cond.duration_pitch = pred = encoders.DurationPitchPredictor(dim=128, dim_hidden=128, depth=1, heads=2)
    red = parallel.GradReducer(coalesce_below=4096)
    cond.grad_reducer = red
    assert pred.grad_reducer is red
    _stand_ins(pred, rank)
    x = torch.zeros(2, 3, 128, requires_grad=True)
    prompts = torch.zeros(2, 5, 128, requires_grad=True)
    dur, pitch = encoders._EncoderFunction.apply(pred, pred.grad_reducer, x, prompts, *pred.parameters())
    dur.sum().backward()                                   # only the duration output is used
    named = list(pred.named_parameters())
    ok = all((p.grad is None) if n.startswith("to_pitch_pred.") else torch.allclose(p.grad, torch.full(p.shape, 1.5 * (i + 1)))
             for i, (n, p) in enumerate(named))
    ok &= bool((x.grad == 3.0).all()) and bool((prompts.grad == 4.0).all())
    q.put((rank, ok, red.bytes_reduced))
    dist.destroy_process_group()


def test_predictor_gradients_are_averaged_over_ranks_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35600 + os.getpid() % 2000
    procs = [ctx.Process(target=_predictor_reducer_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, ok, nbytes in res:
        assert ok and nbytes > 0
