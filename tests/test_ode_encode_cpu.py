"""CPU checks of the latent-interpolation routes: the reference's three noise edits (trainers/interpolate_latent.py:23-57)
against tests/golden/ode_encode.npz (made by the unmodified reference, tests/golden/make_golden_ode_encode.py), and the
import aliases of the two interpolation trainers."""
import os

import numpy as np
import torch

G = os.path.join(os.path.dirname(__file__), "golden")


def test_noise_edits_match_the_reference_exactly():
    from lion_b200.trainers.interpolate_latent import interpolate_noise, linear_interpolate_noise, subtract_noise
    z = np.load(os.path.join(G, "ode_encode.npz"))
    for fn, key in ((interpolate_noise, "n_interpolate"), (linear_interpolate_noise, "n_linear"), (subtract_noise, "n_subtract")):
        noise = torch.from_numpy(z["n_in"]).clone()
        out = fn(noise)
        assert out is noise, "%s edits its argument in place and returns it" % fn.__name__
        assert torch.equal(out, torch.from_numpy(z[key])), fn.__name__


def test_alias_table_resolves_the_interpolation_trainers():
    import importlib
    import lion_b200
    for ref_name in ("trainers.interpolate_latent", "trainers.encode_interp_interp"):
        mod = importlib.import_module(lion_b200._ALIASES[ref_name])
        assert hasattr(mod, "Trainer"), ref_name
    from lion_b200.trainers import encode_interp_interp, interpolate_latent
    assert hasattr(interpolate_latent, "generate_samples") and hasattr(encode_interp_interp.Trainer, "eval_nll")
