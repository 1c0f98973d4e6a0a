"""GPU: the sampler's captured steps live in the model's one graph cache (`Model._captured`).  A step captured on a
workspace leaves the cache with that workspace, so sampling that shape again captures anew instead of replaying into
memory the workspace no longer owns; and `invalidate_packed()` after a `.data` update reaches the sampler's graphs."""
import pytest
import torch

from helpers import build_model, load_model_golden

pytestmark = pytest.mark.gpu


def _case(mode, seed_offset=0):
    """(model, sample kwargs, forward kwargs) of the unconditional model, or of the conditional one guided at scale 2."""
    z, kwargs, seed = load_model_golden("uncond_small" if mode == "uncond" else "cond_small")
    model = build_model(kwargs, seed + seed_offset, device="cuda")
    if mode == "uncond":
        return model, {}, {}
    prompt, cond = torch.from_numpy(z["in_prompt"]).cuda(), torch.from_numpy(z["in_cond"]).cuda()
    return model, dict(prompt_enc=prompt, cond=cond, cond_scale=2.0), dict(prompt=prompt, cond=cond, cond_drop_prob=0.)


def _sampler(model, graphs):
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    return NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, cuda_graphs=graphs)


@pytest.mark.parametrize("mode", ["uncond", "cfg"])
def test_sampler_graph_leaves_the_cache_with_its_workspace(mode, monkeypatch):
    from naturalspeech2_pytorch_b200 import model as model_module
    captures, capture = [], model_module._capture

    def counted(step):
        captures.append(1)
        return capture(step)
    monkeypatch.setattr(model_module, "_capture", counted)
    model, kw, fwd = _case(mode)
    model.max_cached_shapes = 2
    A = 64
    noise = torch.randn(2, A, 128, generator=torch.Generator().manual_seed(5))
    run = lambda sampler: sampler.sample(length=A, batch_size=2, noise=noise, **kw)  # noqa: E731
    ref = run(_sampler(model, False))
    ns = _sampler(model, True)
    assert torch.equal(run(ns), ref) and len(captures) == 1
    [(key, entry)] = model._graphs.items()
    ws_a = entry["ws_key"]
    shapes = [(t.shape, t.dtype) for t in model._ws[ws_a].values()]
    del entry
    for n in (96, 128):   # eager forwards at two other lengths push workspace A out of the LRU
        model(torch.randn(2, n, 128, device="cuda"), torch.rand(2, device="cuda"), **fwd)
    assert ws_a not in model._ws
    assert key not in model._graphs
    assert all(e["ws_key"] in model._ws for e in model._graphs.values()), "an entry outlived its workspace"
    # memory handed out after the eviction, of the evicted workspace's sizes: a replay of the old graph would write it
    sentinels = [torch.full(s, 7.0, dtype=dt, device="cuda") for s, dt in shapes]
    assert torch.equal(run(ns), ref)
    assert len(captures) == 2 and key in model._graphs
    torch.cuda.synchronize()
    assert all(bool((t == 7.0).all()) for t in sentinels), "a replay wrote into memory it does not own"


@pytest.mark.parametrize("mode", ["uncond", "cfg"])
def test_data_updates_need_invalidate_packed(mode):
    """`.data` updates (EMA-style lerp_) do not bump the version counter: `invalidate_packed()` makes them visible to
    the sampler's captured graphs too."""
    m1, kw, _ = _case(mode)
    m2, _, _ = _case(mode, seed_offset=1)
    noise = torch.randn(2, 160, 128, generator=torch.Generator().manual_seed(6))
    run = lambda sampler: sampler.sample(length=160, batch_size=2, noise=noise, **kw)  # noqa: E731
    ns = _sampler(m1, True)
    before = run(ns)
    with torch.no_grad():
        for p, q in zip(m1.parameters(), m2.parameters()):
            p.data.copy_(q.data)
    m1.invalidate_packed()
    after = run(ns)
    assert torch.equal(after, run(_sampler(m2, False))) and not torch.equal(after, before)
