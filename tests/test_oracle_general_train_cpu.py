"""The oracle's training step of the general multi-light model (three SG sets in ``lgtSGs_list``, outside the
state_dict) against the real reference's, recorded by tests/golden/make_general_train_golden.py on general_g20.pt's
state: relight steps with mixed light ids and without light 1, and a phase-1 (radiance-only) step.  Same seed => same
random stream, so maps and loss are bit-exact and every gradient, each SG set's included, agrees to 1e-6."""
import pytest
import torch

from oracle import tensoir_oracle as O
from gpu_helpers import load_fixture
from helpers import oracle_field, named_oracle_params

RUNS = ("relight_mixed", "relight_no1", "phase1")


@pytest.fixture(scope="module")
def train_fx():
    return load_fixture("general_g20_train.pt")


def train_loss(ret, is_relight):
    """make_general_train_golden.train_loss."""
    target = torch.full_like(ret["rgb_map"], 0.5)
    loss = ((ret["rgb_map"] - target) ** 2).mean()
    if is_relight:
        loss = (loss + 0.2 * ((ret["rgb_with_brdf_map"] - target) ** 2).mean()
                + 0.0005 * ret["normals_diff_map"].mean() + 0.001 * ret["normals_orientation_loss_map"].mean()
                + 0.001 * ret["albedo_smoothness_loss"] + 0.001 * ret["roughness_smoothness_loss"])
    return loss


def general_params(f):
    """reference parameter name -> oracle tensor, with each light's SG set as ``lgtSGs_list.k``."""
    return named_oracle_params(f) | {f"lgtSGs_list.{k}": t for k, t in enumerate(f.lgt_sgs)}


@pytest.mark.parametrize("name", RUNS)
def test_general_train_step_matches_reference(golden_general, train_fx, name):
    run = train_fx["runs"][name]
    want_grads = train_fx[name]
    f = oracle_field(golden_general, requires_grad=True)
    torch.manual_seed(run["seed"])
    got = O.renderer_train(f, train_fx["rays"], run["light_idx"], train_fx["n_samples"], True, True,
                           run["is_relight"], 'stratified_sampling', 160000, train_fx["second_nsample"])
    assert got.keys() == run["maps"].keys()
    for k, w in run["maps"].items():
        if w is None:
            assert got[k] is None, k
        elif w.dtype == torch.bool:
            assert torch.equal(got[k], w), k
        else:
            assert torch.equal(got[k].detach(), w), (k, float((got[k].detach() - w).abs().max()))
    assert int(run["maps"]["acc_map"].gt(0.5).sum()) > 20          # most rays hit: the secondary path runs
    loss = train_loss(got, run["is_relight"])
    assert torch.equal(loss.detach(), run["loss"])
    loss.backward()
    params = general_params(f)
    assert set(params) == set(want_grads), set(params) ^ set(want_grads)
    for k, w in want_grads.items():
        g = params[k].grad
        if w is None:
            assert g is None or float(g.abs().max()) == 0.0, k
            continue
        assert torch.allclose(g, w, rtol=1e-6, atol=1e-6), (k, float((g - w).abs().max()))
    ids = set(run["light_idx"].view(-1).tolist())
    sg = [f"lgtSGs_list.{k}" for k in range(3)]
    if run["is_relight"]:
        for k in range(3):
            # a light outside the batch gets an exactly zero SG gradient; one inside it a nonzero one
            assert (float(want_grads[sg[k]].abs().max()) > 0) == (k in ids), (k, ids)
            assert (float(params[sg[k]].grad.abs().max()) > 0) == (k in ids), (k, ids)
        # every light_line row has a gradient: the intrinsic feature reads the mean of all rows
        # (tensoRF_general_multi_lights.py:160-161)
        assert bool((want_grads["light_line.weight"].abs().amax(1) > 0).all())
    else:
        assert all(want_grads[k] is None for k in sg)
        assert want_grads["light_line.weight"] is not None
