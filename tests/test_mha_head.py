"""MN with head_type='multihead_attention_pooling', CPU side: the module tree against the reference's state_dict and
parameter order, the fp64 oracle of the head (tests/mha_util.py on oracle/net_oracle.py) against the golden vectors of
the unmodified reference (tests/golden/make_golden_mha.py), the heads that still raise, and the argument checks of the
head's C-ABI entry points (fake pointers: every check precedes any launch)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.mha_util import CASES, HEAD, build_mha_model, case_inputs, mn_mha_forward
from tests.util import GOLDEN, fmap_digest, golden

torch.set_num_threads(8)


@pytest.fixture(scope="module")
def g():
    return golden("mn_mha")


def test_golden_attention_is_far_from_uniform(g):
    """the golden state makes the attention matter: for most (b, h, k) max / min of the normalised attention over t is
    at least 1.5, in eval and in training"""
    for case in CASES:
        assert g[case + "__eval_att_far"] >= 0.8, case
        assert g[case + "__train_att_far"] >= 0.8, case


def test_state_dict_and_parameter_order_match_reference(g):
    want = json.load(open(os.path.join(GOLDEN, "statedict_mn04_mha.json")))
    m = build_mha_model("mn04_h4")
    got = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert list(got) == list(want) and got == want
    for case in CASES:
        names = [n for n, _ in build_mha_model(case).named_parameters()]
        assert names == [str(s) for s in g[case + "__grad_names"]], case
    assert names[-3:] == ["classifier.head_weight", "classifier.subspace_proj.weight", "classifier.subspace_proj.bias"]


def test_construction_uses_the_rng_like_the_reference():
    """the reference's initialisation (Linear N(0, 0.01), zero bias, head_weight = 1/H) and attributes; calling the
    container directly raises (the engine runs it).  That construction draws from the RNG exactly as the reference does
    (so a seeded script draws the same batches) is what the script test on the GPU relies on: both sides start there."""
    from efficientat_b200.models.mn.model import get_model
    torch.manual_seed(0)
    m = get_model(width_mult=0.4, head_type=HEAD, multihead_attention_heads=3, verbose=False)
    head = m.classifier
    assert torch.equal(head.head_weight, torch.full((1, 3, 1), 1.0 / 3))
    assert head.subspace_proj.bias.abs().max() == 0
    assert abs(head.subspace_proj.weight.std().item() - 0.01) < 1e-3
    assert head.num_heads == 3 and head.out_dim == 527 and head.epsilon == 1e-7
    with pytest.raises(RuntimeError, match="parameter container"):
        head(torch.zeros(1, 384, 4, 7))


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_head_matches_reference_vectors(g, case):
    """fp64 oracle against the reference run in fp32 (CPU): eval logits 1e-4, features 2e-4, feature maps 1e-3 of the
    largest digest entry; training-step logits 1e-4, loss 1e-6, every gradient norm 1e-3 relative"""
    width, _, _, H, K = CASES[case]
    m = build_mha_model(case, golden=g)
    sd = {k: v.detach().clone().double() for k, v in m.state_dict().items()}
    spec, y = case_inputs(case)
    with torch.no_grad():
        logits, feat, fmaps = mn_mha_forward(sd, spec.double(), width, H, K, return_fmaps=True)
    assert np.abs(logits.numpy() - g[case + "__eval_logits"]).max() < 1e-4
    assert np.abs(feat.numpy() - g[case + "__eval_feat"]).max() < 2e-4
    d, want = fmap_digest(fmaps), g[case + "__eval_fmaps"]
    assert np.abs(d - want).max() < 1e-3 * max(1.0, np.abs(want).max())
    names = [n for n, _ in m.named_parameters()]
    for n in names:
        sd[n].requires_grad_(True)
    lt, _ = mn_mha_forward(sd, spec.double(), width, H, K, training=True)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(lt, y.double())
    loss.backward()
    assert np.abs(lt.detach().numpy() - g[case + "__train_logits"]).max() < 1e-4
    assert abs(loss.item() - float(g[case + "__train_loss"])) < 1e-6
    gn = np.array([sd[n].grad.norm().item() for n in names])
    rel = np.abs(gn - g[case + "__grad_norm"]) / np.maximum(g[case + "__grad_norm"], 1e-9)
    bad = [(n, r) for n, r, ref in zip(names, rel, g[case + "__grad_norm"]) if r > 1e-3 and ref > 1e-6]
    assert not bad, bad[:10]


def test_unsupported_heads_still_raise():
    """DyMN has no attention head (dymn/model.py:140-142); the fully-convolutional head is not implemented for either"""
    from efficientat_b200.models.dymn.model import dymn
    from efficientat_b200.models.mn.model import get_model as mn
    for head in (HEAD, "fully_convolutional"):
        with pytest.raises(NotImplementedError):
            dymn(width_mult=0.4, head_type=head)
    with pytest.raises(NotImplementedError):
        mn(width_mult=0.4, head_type="fully_convolutional", verbose=False)
    with pytest.raises(NotImplementedError, match="unknown"):
        mn(width_mult=0.4, head_type="attention", verbose=False)


def test_pretrained_loading_raises_like_the_reference(monkeypatch):
    """the released checkpoints have the 'mlp' head; the reference then looks up 'classifier.1.bias' and raises KeyError
    (mn/model.py:287-302) -- so does this factory, instead of loading the trunk silently"""
    from efficientat_b200.models.mn import model as M
    sd = M.get_model(width_mult=0.4, verbose=False).state_dict()
    monkeypatch.setattr(M, "load_state_dict_from_url", lambda *a, **k: {k: v.clone() for k, v in sd.items()})
    with pytest.raises(KeyError, match="classifier.1.bias"):
        M.get_model(width_mult=0.4, pretrained_name="mn04_as", head_type=HEAD, verbose=False)
    M.get_model(width_mult=0.4, pretrained_name="mn04_as", verbose=False)        # the 'mlp' head still loads


def test_head_entry_points_reject_bad_arguments_before_any_launch():
    from efficientat_b200._lib import EatError, lib
    L = lib()
    fake = 4096                                                   # never dereferenced: validation comes first
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.freq_pool(fake, 0, 0, 0, 0, fake, fake, 2, 4, 7, 10, 0)          # fp32, C = 10
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.freq_pool(fake, 1, 0, 0, 0, fake, fake, 2, 4, 7, 12, 0)          # bf16, C = 12
    with pytest.raises(EatError, match="F, T, C >= 1"):
        L.freq_pool(fake, 0, 0, 0, 0, fake, fake, 2, 4, 0, 16, 0)
    with pytest.raises(EatError, match="scale and shift"):
        L.freq_pool(fake, 0, fake, 0, 2, fake, fake, 2, 4, 7, 16, 0)
    with pytest.raises(EatError, match="dtype"):
        L.freq_pool(fake, 2, 0, 0, 0, fake, fake, 2, 4, 7, 16, 0)
    with pytest.raises(EatError, match="aligned"):
        L.freq_pool(fake + 4, 0, 0, 0, 0, fake, fake, 2, 4, 7, 16, 0)
    with pytest.raises(EatError, match="required"):
        L.freq_pool(0, 0, 0, 0, 0, fake, fake, 2, 4, 7, 16, 0)
    with pytest.raises(EatError, match="multiple of the vector width"):
        L.freq_pool_bwd(fake, 0.25, fake, 1, 2, 4, 7, 20, 0)
    with pytest.raises(EatError, match="aligned"):
        L.freq_pool_bwd(fake, 0.25, fake + 8, 0, 2, 4, 7, 16, 0)
    with pytest.raises(EatError, match="T, H, K >= 1"):
        L.att_pool_fwd(fake, fake, 1e-7, fake, 0, 0, 2, 0, 4, 527, 0)
    with pytest.raises(EatError, match="T, H, K >= 1"):
        L.att_pool_fwd(fake, fake, 1e-7, fake, 0, 0, 2, 7, 0, 527, 0)
    with pytest.raises(EatError, match="eps"):
        L.att_pool_fwd(fake, fake, 0.0, fake, 0, 0, 2, 7, 4, 527, 0)
    with pytest.raises(EatError, match="go together"):
        L.att_pool_fwd(fake, fake, 1e-7, fake, fake, 0, 2, 7, 4, 527, 0)
    with pytest.raises(EatError, match="required"):
        L.att_pool_fwd(0, fake, 1e-7, fake, 0, 0, 2, 7, 4, 527, 0)
    with pytest.raises(EatError, match="T, H, K >= 1"):
        L.att_pool_bwd(fake, fake, fake, fake, fake, fake, 1e-7, fake, fake, 2, 7, 4, 0, 0)
    with pytest.raises(EatError, match="every pointer"):
        L.att_pool_bwd(fake, fake, fake, fake, 0, fake, 1e-7, fake, fake, 2, 7, 4, 527, 0)
    # empty batches are a no-op, not an error
    L.freq_pool(0, 0, 0, 0, 0, 0, 0, 0, 4, 7, 16, 0)
    L.freq_pool_bwd(0, 0.25, 0, 0, 0, 4, 7, 16, 0)
    L.att_pool_fwd(0, 0, 1e-7, 0, 0, 0, 0, 7, 4, 527, 0)
    L.att_pool_bwd(0, 0, 0, 0, 0, 0, 1e-7, 0, 0, 0, 7, 4, 527, 0)
