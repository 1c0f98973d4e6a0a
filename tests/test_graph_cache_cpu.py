"""The model's one cache of captured CUDA graphs (`Model._captured`), on CPU: which entries leave it when a workspace is
evicted, on a repack and past the LRU bound, for the model's own steps and the sampler's alike, and when the static
conditioning is refreshed.  A CPU model packs its weights and allocates CPU workspaces; only the capture itself is
replaced, by a placeholder."""
import pytest
import torch

from naturalspeech2_pytorch_b200 import Model, model as model_module
from naturalspeech2_pytorch_b200.model import Conditioning

CPU = torch.device("cpu")


@pytest.fixture
def model(monkeypatch):
    monkeypatch.setattr(model_module, "_capture", lambda step: "graph")
    torch.manual_seed(0)
    m = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1)
    m.max_cached_shapes = 2
    return m


def _model_key(N, p=0.):
    return (1, N, p, None, False, "cpu")


def _sampler_key(N, cond_scale=None):
    return ("sample", (1, N, 128), None, cond_scale, "v", False, "cpu")


def _put(m, key, N, conditioning=None):
    """An entry captured on the (1, N) workspace, inserted the way the model's and the sampler's steps are."""
    m._workspace(1, N, CPU)
    return m._captured(key, m._ws_key(1, N, CPU), conditioning, lambda cond: ({"buf": torch.zeros(1)}, None))


def test_evicting_a_workspace_drops_the_entries_captured_on_it(model):
    _put(model, _model_key(16), 16)
    _put(model, _sampler_key(16), 16)
    _put(model, _model_key(32), 32)
    assert list(model._ws) == [(1, 16, "cpu"), (1, 32, "cpu")]
    model._workspace(1, 48, CPU)   # evicts (1, 16): both steps captured on it leave, the one on (1, 32) stays
    assert list(model._graphs) == [_model_key(32)]
    assert all(e["ws_key"] in model._ws for e in model._graphs.values())
    model._workspace(1, 32, CPU)
    model._workspace(1, 64, CPU)   # evicts (1, 48), on which nothing was captured
    assert list(model._graphs) == [_model_key(32)]
    assert list(model._ws) == [(1, 32, "cpu"), (1, 64, "cpu")]


def _bump_a_parameter(m):
    with torch.no_grad():
        next(m.parameters()).add_(1.0)   # moves the version counter, like an optimizer step


@pytest.mark.parametrize("repack", [lambda m: m.invalidate_packed(), lambda m: m.to(CPU), _bump_a_parameter],
                         ids=["invalidate_packed", "to", "parameter_version"])
def test_a_repack_drops_every_entry(model, repack):
    _put(model, _model_key(16), 16)
    _put(model, _sampler_key(32), 32)
    repack(model)
    _put(model, _sampler_key(16), 16)
    assert list(model._graphs) == [_sampler_key(16)]


def test_one_lru_bound_over_model_and_sampler_entries(model):
    keys = [_model_key(16, 0.), _sampler_key(16), _model_key(16, 1.), _sampler_key(16, 3.)]
    for k in keys:
        _put(model, k, 16)
    assert list(model._graphs) == keys   # 2 * max_cached_shapes
    _put(model, keys[0], 16)             # a hit: now the most recent
    _put(model, _sampler_key(16, 2.), 16)
    assert list(model._graphs) == keys[2:] + [keys[0], _sampler_key(16, 2.)]
    _put(model, _model_key(32), 32)
    assert len(model._graphs) == 2 * model.max_cached_shapes and keys[2] not in model._graphs


def test_static_conditioning_is_refreshed_when_another_object_arrives(model):
    c1 = Conditioning(tokens=torch.zeros(3), length=16)
    entry = _put(model, _sampler_key(16), 16, c1)
    assert entry["cond"]["tokens"] is not c1["tokens"] and torch.equal(entry["cond"]["tokens"], c1["tokens"])
    c1["tokens"].fill_(1.)   # the same object again: its copy is not refreshed
    assert torch.equal(_put(model, _sampler_key(16), 16, c1)["cond"]["tokens"], torch.zeros(3))
    c2 = Conditioning(tokens=torch.full((3,), 2.), length=16)
    assert torch.equal(_put(model, _sampler_key(16), 16, c2)["cond"]["tokens"], c2["tokens"])
