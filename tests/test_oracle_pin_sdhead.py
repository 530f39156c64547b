"""Pins the diffusion-loss restatement (oracle/unet_oracle.py `diffusion_loss`, `add_noise`, and the CFG-dropout row mix) to the
reference code: `StableDiffusionHead._compute_snr` and `.forward` (modeling_plugins.py:468-577), exec'd verbatim on CPU with stand-in
`vae` / `noise_scheduler` / `projector` / `unet` objects built from the oracle's modules (oracle/plugin_scenarios.py) by
`python -m oracle.gen_golden_plugins`; their losses are stored in tests/golden/plugins.npz.  Same seed => the reference's own RNG draws
(randn_like, randn, randint, bernoulli — in its order) are reproduced and fed to the restatement, so every branch (`noise_offset`,
`input_perturbation`, `snr_gamma`, `drop_prob`) is compared to the reference's arithmetic.  What stays from-spec is only the inside of
diffusers' UNet / VAE / scheduler classes (DESIGN.md §2)."""
import os

import numpy as np
import pytest
import torch

from oracle import plugin_scenarios as PS

GOLD = os.path.join(os.path.dirname(__file__), "golden", "plugins.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.mark.parametrize("noise_offset,input_perturbation,snr_gamma,drop_prob", PS.SDHEAD_CASES)
def test_diffusion_loss_restatement_equals_live_reference_forward(gold, noise_offset, input_perturbation, snr_gamma, drop_prob):
    i = PS.SDHEAD_CASES.index((noise_offset, input_perturbation, snr_gamma, drop_prob))
    got = PS.oracle_sdhead(noise_offset, input_perturbation, snr_gamma, drop_prob)
    torch.testing.assert_close(float(got), float(gold[f"sdhead_{i}"]), rtol=1e-6, atol=1e-7)


def test_dummy_forward_of_the_reference_is_a_zero(gold):
    """(:500-509) the reference's images=None branch only feeds DDP's unused-parameter check; our reducer needs no such pass."""
    assert float(gold["sdhead_dummy"]) == 0.0
