"""The training fixtures (tests/golden/train_*.npz) on the CPU: fp64 autograd of the oracle functions
(oracle/interaction_oracle.py) reproduces the reference classes' gradients at the interaction stage's inputs and
parameters, which is what pins the oracle's backward; the fixtures' parameter names are the drop-in classes'; and, where
the reference is mounted, a training family regenerates bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ranker_training_cases as T
from conftest import GOLDEN_DIR, ROOT
from oracle import interaction_oracle as O
from oracle import make_golden as M
from oracle import reference_loader as R

# the generator checks the oracle's backward to 1e-10 on the fp64 values; the fixtures store them rounded to fp32, so
# here the oracle runs on the rounded interaction inputs
PIN = 1e-5


def _leaf(t):
    return t.double().clone().requires_grad_(True)


def _pin(got, ref, what):
    ref = ref.double()
    err = (got.detach() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= PIN * scale, f"{what}: oracle backward {err / scale:.2e} off the reference's"


def _kernel_pool_pin(name, g):
    sd = T.state_dict(g)
    qm, dm = g["q_mask"].double(), g["d_mask"].double()
    gs = g["gout__score"].double()
    if name == "train_knrm":
        q, d, w = _leaf(g["q"]), _leaf(g["d"]), _leaf(sd["dense.weight"].view(-1))
        K = int(g["cfg"][0])
        s, _ = O.kernel_pool_knrm(q, d, qm, dm, torch.tensor(O.knrm_kernel_mus(K), dtype=torch.float32).double(),
                                  torch.tensor(O.knrm_kernel_sigmas(K), dtype=torch.float32).double(), w)
        s.backward(gs)
        return s, {"gi__q": q.grad, "gi__d": d.grad, "gp__dense.weight": w.grad.view(1, -1)}
    if name == "train_conv_knrm":
        n, K = int(g["cfg"][1]), int(g["cfg"][2])
        qg = [_leaf(g[f"ctx__qg{i}"].transpose(1, 2)) for i in range(n)]
        dg = [_leaf(g[f"ctx__dg{i}"].transpose(1, 2)) for i in range(n)]
        w = _leaf(sd["dense.weight"].view(-1))
        s, _ = O.conv_knrm_cross_match(qg, dg, qm, dm, torch.tensor(O.knrm_kernel_mus(K), dtype=torch.float32).double(),
                                       torch.tensor(O.knrm_kernel_sigmas(K), dtype=torch.float32).double(), w)
        s.backward(gs)
        grads = {"gp__dense.weight": w.grad.view(1, -1)}
        for i in range(n):
            grads[f"gctx__qg{i}"] = qg[i].grad.transpose(1, 2)
            grads[f"gctx__dg{i}"] = dg[i].grad.transpose(1, 2)
        return s, grads
    q, d = _leaf(g["ctx__q_ctx"]), _leaf(g["ctx__d_ctx"])
    w, a = _leaf(sd["kernel_bin_weights.weight"].view(-1)), _leaf(sd["kernel_alpha_scaler"].view(-1))
    mu, sigma = sd["mu"].view(-1).double(), sd["sigma"].view(-1).double()
    grads = {}
    if name == "train_tk_sparse":
        gate = _leaf(g["ctx__gate"].squeeze(1))
        s, _ = O.kernel_pool_tk_sparse(q, d, qm, dm, gate, mu, sigma, a, w)
        s.backward(gs)
        # the gate is the ranker's second output too: its gradient adds that output's upstream gradient
        grads["gctx__gate"] = (gate.grad + g["gout__document_stop_words"].squeeze(1).double()).unsqueeze(1)
    else:
        s, _ = O.kernel_pool_tk(q, d, qm, dm, mu, sigma, a, w)
        s.backward(gs)
    grads.update({"gctx__q_ctx": q.grad, "gctx__d_ctx": d.grad, "gp__kernel_bin_weights.weight": w.grad.view(1, -1),
                  "gp__kernel_alpha_scaler": a.grad.view(1, 1, -1)})
    return s, grads


def _tkl_pin(name, g):
    sat = name[len("train_tkl_"):]
    sd = T.state_dict(g)
    q, c = _leaf(g["ctx__q_ctx"]), _leaf(g["ctx__doc_chunks_ctx"])
    leaf = {"dense_weight": _leaf(sd["dense.weight"].view(-1)), "chunk_scoring": _leaf(sd["chunk_scoring"].view(-1)),
            "sat_emb_reduce1_weight": _leaf(sd["sat_emb_reduce1.weight"].view(-1)),
            "kernel_mult0": _leaf(sd["kernel_mult"][0].reshape(-1))}
    for k in ("sat_normer.weight", "sat_normer.bias", "saturation_linear.weight", "saturation_linear.bias",
              "saturation_linear2.weight", "saturation_linear2.bias", "saturation_linear3.weight", "saturation_linear3.bias"):
        leaf[k.replace(".", "_")] = _leaf(sd[k].view(-1))
    params = dict(leaf, mu=sd["mu"].double(), sigma=sd["sigma"].double())
    s, sec = O.tkl_interaction(q, g["q_mask"].double(), c, g["doc_chunk_mask"].double(), g["packed_indices"],
                               int(g["chunk_pieces"]), params, sat)
    assert torch.equal(sec["top_non_overlapping_idx"], g["top_non_overlapping_idx"])
    s.backward(g["gout__score"].double())
    grads = {"gctx__q_ctx": q.grad, "gctx__doc_chunks_ctx": c.grad,
             "gp__dense.weight": leaf["dense_weight"].grad.view(1, -1),
             "gp__chunk_scoring": leaf["chunk_scoring"].grad.view(1, -1)}
    if sat == "embedding":
        grads["gp__sat_emb_reduce1.weight"] = leaf["sat_emb_reduce1_weight"].grad.view(1, -1)
        for k in ("sat_normer.weight", "sat_normer.bias", "saturation_linear.weight", "saturation_linear.bias",
                  "saturation_linear2.weight", "saturation_linear2.bias", "saturation_linear3.weight",
                  "saturation_linear3.bias"):
            grads["gp__" + k] = leaf[k.replace(".", "_")].grad.view_as(sd[k])
    else:
        km = torch.zeros_like(sd["kernel_mult"], dtype=torch.float64)
        km[0] = leaf["kernel_mult0"].grad.view_as(km[0])
        grads["gp__kernel_mult"] = km
    return s, grads


@pytest.mark.parametrize("name", T.KERNEL_POOLING + T.TKL)
def test_oracle_backward_is_the_reference_backward(name):
    g = T.load(name)
    s, grads = (_tkl_pin if name in T.TKL else _kernel_pool_pin)(name, g)
    _pin(s, g["out__score"], f"{name} score")
    for k, v in grads.items():
        _pin(v, g[k], f"{name} {k}")
    # every gradient at the interaction stage's inputs is covered
    assert {k for k in g if k.startswith("gctx__")} <= set(grads)


def test_colbert_and_bert_dot_oracle_backward():
    g = T.load("train_colbert")
    for key, prefix in (("score", ""), ("allpairs", "ib_")):
        q, d = _leaf(g["q"]), _leaf(g["d"])
        if key == "score":
            out = O.maxsim_pairs(q, d, g["q_mask"], g["d_mask"])
        else:
            out = O.maxsim_allpairs(q, g["q_mask"], d, g["d_mask"])
        out.backward(g["gout__" + key].double())
        _pin(out, g["out__" + key], f"colbert {key}")
        _pin(q.grad, g[f"gi__{prefix}q"], f"colbert {key} grad q")
        _pin(d.grad, g[f"gi__{prefix}d"], f"colbert {key} grad d")
    g = T.load("train_bert_dot")
    q, d = _leaf(g["qv"]), _leaf(g["dv"])
    s = O.dot_pairs(q, d)
    s.backward(g["gout__score"].double())
    _pin(s, g["out__score"], "bert_dot score")
    _pin(q.grad, g["gi__qv"], "bert_dot grad qv")
    _pin(d.grad, g["gi__dv"], "bert_dot grad dv")


@pytest.mark.parametrize("name", T.WITH_PARAMETERS)
def test_fixture_parameters_are_the_drop_in_parameters(name):
    """Names (in order) and shapes of the fixture's parameters are the drop-in class's, and every parameter either has
    a stored gradient or is listed as receiving none."""
    g = T.load(name)
    m = T.build(name, g)
    names = [n for n, _ in m.named_parameters()]
    assert names == g["param_names"]
    no_grad = set(g["no_grad_params"])
    for n, p in m.named_parameters():
        assert (n in no_grad) != (("gp__" + n) in g), n
        if n not in no_grad and n not in T.TKL_TRIMMED:
            assert g["gp__" + n].shape == p.shape, n


def test_tkl_parameters_without_gradient():
    """The TKL parameters the reference's backward never reaches, per saturation mode."""
    common = {"mu", "sigma", "mixer_sat", "mixer_end"}
    sat_embedding = {"sat_normer.weight", "sat_normer.bias", "sat_emb_reduce1.weight"} | {
        f"saturation_linear{i}.{w}" for i in ("", "2", "3") for w in ("weight", "bias")}
    assert set(T.load("train_tkl_embedding")["no_grad_params"]) == common | {"kernel_mult"}
    assert set(T.load("train_tkl_log")["no_grad_params"]) == common | sat_embedding


@pytest.mark.skipif(not R.reference_available(), reason="reference repo not mounted (GPU box)")
@pytest.mark.parametrize("family", [name for name, _ in M.TRAINING_FAMILIES])
def test_training_fixture_regenerates_from_reference(family, tmp_path):
    """Re-run a training family from the reference classes into a scratch directory and compare with the committed
    fixtures, array by array, bit for bit."""
    code = ("import sys; from oracle import make_golden as M; M.GOLDEN_DIR = sys.argv[1]; "
            f"sys.argv = ['make_golden', '{family}']; sys.exit(M.main())")
    res = subprocess.run([sys.executable, "-c", code, str(tmp_path)], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    written = sorted(os.listdir(tmp_path))
    assert written and all(f.startswith(family) for f in written), written
    for f in written:
        new = np.load(os.path.join(tmp_path, f))
        old = np.load(os.path.join(GOLDEN_DIR, f))
        assert sorted(new.files) == sorted(old.files), f
        for k in old.files:
            assert np.array_equal(new[k], old[k]), f"{f}: {k}"
