"""CPU: the duration / pitch predictor's dropout plumbing - which sites draw (pinned to the reference module's own
nn.Dropout / Attend probabilities), their site numbers, the seed draw and the Conditioner flags."""
import sys
from pathlib import Path

import pytest
import torch
from torch import nn

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

KW = dict(dim=128, dim_hidden=128, depth=2, heads=2, dropout=0.3)


def test_dropout_probabilities_match_the_reference_module():
    """Every nn.Dropout of the reference's DurationPitchPredictor, read from the module itself: the Blocks' (after the
    SiLU) have p = 0 - the trunk builds its ResnetBlocks without a dropout argument - and only the cross attentions'
    Attend carries `dropout`.  Ours draws at exactly those sites with the same p."""
    ns2 = bench.import_reference()
    if ns2 is None:
        pytest.skip("oracle/_ref (pip-installed reference) is not present")
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor
    ref = ns2.DurationPitchPredictor(**KW)
    ours = DurationPitchPredictor(**KW)
    block, attn, other = [], [], []
    for name, m in ref.named_modules():
        if isinstance(m, nn.Dropout):
            (block if ".blocks." in name else attn if name.endswith("attend.attn_dropout") else other).append(m.p)
        if type(m).__name__ == "Attend":
            assert m.dropout == ours.attn_dropout, name
    assert not other
    assert len(block) == 2 * 2 * 3 * 2 and len(attn) == 2 * 2          # trunks x depth x ResnetBlocks x Blocks
    assert set(block) == {ours.conv_dropout} == {0.0}
    assert set(attn) == {ours.attn_dropout} == {0.3}


def test_attention_sites_are_distinct_and_in_forward_order():
    """Cross attention of layer l of trunk t (0 duration - the forward runs it first - and 1 pitch) is site t depth + l."""
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor
    m = DurationPitchPredictor(dim=512)
    assert (m.attn_dropout, m.conv_dropout, m.train_dropout) == (0.2, 0.0, False)   # ns2.py:484
    sites = [m._cross_attn_dropout(5, name, l) for name in ("d", "p") for l in range(10)]
    assert [s[1] for s in sites] == list(range(20)) and {(s[0], s[2]) for s in sites} == {(5, 0.2)}
    assert m._cross_attn_dropout(None, "p", 9) is None


def test_predictor_draws_a_seed_only_when_asked():
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor
    m = DurationPitchPredictor(**KW).train()
    state = torch.get_rng_state()
    assert m._dropout_seed() is None and torch.equal(torch.get_rng_state(), state)   # train_dropout off
    m.train_dropout = True
    torch.manual_seed(4)
    s = m._dropout_seed()
    torch.manual_seed(4)
    assert s == int(torch.randint(0, 2 ** 63 - 1, ())) and 0 <= s < 2 ** 63
    m.eval()
    state = torch.get_rng_state()
    assert m._dropout_seed() is None and torch.equal(torch.get_rng_state(), state)
    z = DurationPitchPredictor(**dict(KW, dropout=0.0)).train()
    z.train_dropout = True
    assert z._dropout_seed() is None                                                   # p = 0 draws nothing
    assert set(z.state_dict()) == set(m.state_dict())                                  # no new parameters or buffers


def test_conditioner_flags():
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    c = Conditioner(num_phoneme_tokens=10)
    assert not c.duration_pitch.train_dropout
    c = Conditioner(num_phoneme_tokens=10, train_dropout=True)
    assert c.prompt_enc.train_dropout and c.phoneme_enc.train_dropout and not c.duration_pitch.train_dropout
    c = Conditioner(num_phoneme_tokens=10, train_duration_pitch=True, duration_pitch_dropout=True)
    assert c.duration_pitch.train_dropout and not c.prompt_enc.train_dropout and not c.phoneme_enc.train_dropout
    assert c.duration_pitch.attn_dropout == 0.2 and c.duration_pitch.conv_dropout == 0.0
