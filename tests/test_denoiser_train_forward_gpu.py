"""GPU: the denoiser's training forward (train mode with gradients: the autograd node of training.DenoiserFunction) is
its inference forward: the output is bit-identical to the eval / no_grad output and the library launches the same
number of kernels, for an unconditional and a conditional model and for condition dropout 0, 1 and 0.5 (the same seed
before each call draws the same two masks, in the reference's order, in both modes)."""
import pytest
import torch

from helpers import build_model, golden_inputs, load_model_golden

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,drop", [("uncond_small", None), ("cond_small", 0.), ("cond_small", 1.),
                                       ("cond_small", 0.5)])
def test_training_forward_is_the_inference_forward(name, drop):
    from naturalspeech2_pytorch_b200 import ops
    z, kwargs, seed = load_model_golden(name)
    model = build_model(kwargs, seed, device="cuda")
    inp = golden_inputs(z, kwargs)
    reps = 4 if drop == 0.5 else 1   # four copies of the batch, so that the two masks disagree on some sample
    x, times = inp["x"].cuda().repeat(reps, 1, 1), inp["times"].cuda().repeat(reps)
    kw = {}
    if kwargs.get("condition_on_prompt"):
        kw = dict(prompt=inp["prompt"].cuda().repeat(reps, 1, 1), cond=inp["cond"].cuda().repeat(reps, 1, 1),
                  cond_drop_prob=drop)

    def forward(train):
        model.train(train)
        torch.manual_seed(123)
        torch.cuda.synchronize()
        before = ops.launch_count()
        with torch.set_grad_enabled(train):
            out = model(x, times, **kw)
        torch.cuda.synchronize()
        return out, ops.launch_count() - before

    forward(False)   # packs the weights
    ref, eval_launches = forward(False)
    out, train_launches = forward(True)
    assert not ref.requires_grad
    assert out.requires_grad and out.grad_fn is not None
    assert torch.equal(out.detach(), ref)
    assert train_launches == eval_launches, (train_launches, eval_launches)
