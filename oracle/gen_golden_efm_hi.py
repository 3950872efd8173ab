"""Generate hierarchical Graph-EFM golden vectors FROM THE REFERENCE SOURCE.

TEST INFRASTRUCTURE ONLY.  Run where the reference source is available:

    python -m oracle.gen_golden_efm_hi

As ``oracle/gen_golden_efm.py`` (same loader, inputs and noise-recording hooks), for the reference ``GraphEFM`` on synthetic
hierarchical graphs: the prior / posterior are ``HiGraphLatentEncoder``s and the latent lives on the top mesh level.  Stored
per case: inputs, state_dict, eps, prior mean / std, prediction (and its std), the posterior's mean / std given a target, and
for ``efm_hi_iso_h64`` the gradients of a scalar loss of prediction and posterior with respect to every parameter at that fixed
eps -> ``tests/golden/efm_hi_cases.*.npz``.
"""
import os
import sys
import tempfile

import numpy as np
import torch
from torch import distributions as tdists

from . import load_reference_efm
from .gen_golden_efm import build_inputs
from .shards import save_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "efm_hi_cases")

# name -> (graph kwargs, datastore kwargs, model kwargs, B, with gradients)
CASES = {
    # (a) the fused path: H = latent = 64, learned isotropic prior; two levels of 81 / 9 nodes
    "efm_hi_iso_h64": (dict(Nx=30, Ny=27, hierarchical=True), dict(d_state=5, d_forcing=6, d_static=1, boundary_width=2),
                       dict(hidden_dim=64, prior_intra_level_layers=1, encoder_intra_level_layers=1,
                            decoder_intra_level_layers=2), 2, True),
    # (b) three levels of 729 / 81 / 9 nodes; diagonal prior, predicted std and output clamping of all three kinds
    "efm_hi_diag_opts_h64": (dict(Nx=84, Ny=82, hierarchical=True), dict(d_state=5, d_forcing=6, d_static=1, boundary_width=3),
                             dict(hidden_dim=64, prior_intra_level_layers=1, encoder_intra_level_layers=1,
                                  decoder_intra_level_layers=2, prior_dist="diagonal", output_std=True,
                                  output_clamping_lower={"var1": -2.5, "var3": -3.0},
                                  output_clamping_upper={"var1": 2.0, "var4": 3.5}), 2, False),
    # (c) constant prior, no intra-level layers (no m2m_embedders), latent_dim != hidden_dim
    "efm_hi_const_h16": (dict(Nx=30, Ny=27, hierarchical=True), dict(d_state=5, d_forcing=6, d_static=1, boundary_width=1),
                         dict(hidden_dim=16, latent_dim=8, learn_prior=False, prior_intra_level_layers=0,
                              encoder_intra_level_layers=0, decoder_intra_level_layers=0), 3, False),
}


def run_case(ref, name, tmp):
    from neural_lam_b200 import synthetic

    gkw, dkw, mkw, B, grads = CASES[name]
    spec = synthetic.make_graph_spec(**gkw)
    ds = synthetic.SyntheticDatastore(spec, **dkw)
    root = os.path.join(tmp, name)
    synthetic.save_graph(spec, os.path.join(root, "graph", "g"))
    stub = load_reference_efm.load_reference.StubDatastore(ds, root)
    torch.manual_seed(42)
    model = ref.GraphEFM(stub, graph_name="g", num_past_forcing_steps=0, num_future_forcing_steps=0, **mkw)
    with torch.no_grad():  # non-trivial LayerNorm affine parameters
        for n_, p_ in model.named_parameters():
            if p_.dim() == 1 and (n_.endswith(".3.weight") or n_.endswith(".3.bias")):
                p_.add_(0.1 * torch.randn_like(p_))
    model.eval()
    x = build_inputs(B, ds.num_grid_nodes, dkw["d_state"], dkw["d_forcing"])
    seen = {}
    prior_forward = model.prior_model.forward

    def record_prior(*a, **k):
        seen["prior"] = prior_forward(*a, **k)
        return seen["prior"]

    model.prior_model.forward = record_prior
    hook = model.decoder.register_forward_pre_hook(lambda mod, args: seen.__setitem__("z", args[1]))
    torch.manual_seed(7)
    with torch.no_grad():
        pred, std = model(x["prev_state"], x["prev_prev_state"], x["forcing"])
        grid_cur = model.embedd_grid_with_target(x["prev_state"], x["prev_prev_state"], x["forcing"], x["target"])
        _, graph_emb = model.embedd_grid_and_graph(x["prev_state"], x["prev_prev_state"], x["forcing"])
        post = model.encoder(grid_cur, graph_emb=graph_emb)
    hook.remove()
    prior = seen["prior"]
    eps = (seen["z"] - prior.mean) / prior.stddev
    blob = {k: v.numpy() for k, v in x.items()}
    blob.update(eps=eps.numpy(), prior_mean=prior.mean.numpy(), prior_std=prior.stddev.numpy(), pred=pred.numpy(),
                post_mean=post.mean.numpy(), post_std=post.stddev.numpy())
    if std is not None:
        blob["pred_std"] = std.numpy()
    for k, v in model.state_dict().items():
        blob["param/" + k] = v.numpy()
    if grads:
        # the same step with eps fixed: the prior's rsample returns mean + eps * std
        class FixedNormal(tdists.Normal):
            def rsample(self, sample_shape=torch.Size()):
                return self.loc + eps * self.scale

        def fixed_prior(*a, **k):
            d = prior_forward(*a, **k)
            return FixedNormal(d.mean, d.stddev)

        model.prior_model.forward = fixed_prior
        g = torch.Generator().manual_seed(5)
        w_pred = torch.randn(pred.shape, generator=g)
        w_post = torch.randn(post.mean.shape, generator=g)
        model.zero_grad()
        pred_g, _ = model(x["prev_state"], x["prev_prev_state"], x["forcing"])
        grid_cur = model.embedd_grid_with_target(x["prev_state"], x["prev_prev_state"], x["forcing"], x["target"])
        _, graph_emb = model.embedd_grid_and_graph(x["prev_state"], x["prev_prev_state"], x["forcing"])
        post_g = model.encoder(grid_cur, graph_emb=graph_emb)
        loss = (pred_g * w_pred).sum() + (post_g.mean * w_post).sum() + (post_g.stddev * w_post).sum()
        loss.backward()
        blob.update(w_pred=w_pred.numpy(), w_post=w_post.numpy(), loss=np.array(loss.item()))
        for k, p_ in model.named_parameters():
            if p_.grad is not None:
                blob["grad/" + k] = p_.grad.numpy()
    model.prior_model.forward = prior_forward
    blob["meta"] = np.array([repr(gkw), repr(dkw), repr(mkw), str(B)]).astype(str)
    n_par = sum(p.numel() for p in model.parameters())
    print(f"  {name}: G={ds.num_grid_nodes} N_top={eps.shape[1]} params={n_par} |pred| max={pred.abs().max():.3f}")
    return blob


def main():
    ref = load_reference_efm.load_efm()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in CASES:
            for k, v in run_case(ref, name, tmp).items():
                out[f"{name}/{k}"] = v
    out["__names__"] = np.array(list(CASES))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    paths = save_shards(OUT, out)
    print(f"wrote {len(paths)} files {OUT}.*.npz")


if __name__ == "__main__":
    sys.exit(main())
