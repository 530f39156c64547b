"""Mint tests/golden/plugins.npz from the REFERENCE'S OWN CODE (build container only: needs /root/reference).

    python -m oracle.gen_golden_plugins

Scenarios and the verbatim exec of the reference methods live in oracle/plugin_scenarios.py.  Stored: the reference's spliced embeddings
(`DreamLLMModel.forward`), conditioning rows / losses (`DreamLLMForCausalMLM.forward`) and diffusion losses (`StableDiffusionHead.forward`,
all six option branches).  tests/test_golden_plugins.py checks the travelling oracles against this file wherever it runs."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import plugin_scenarios as PS  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "plugins.npz")


def main():
    assert PS.reference_available(), "needs /root/reference"
    d = {}
    for i, (n_images, with_dream) in enumerate(PS.SPLICE_CASES):
        out, seen = PS.live_splice(n_images, with_dream)
        d[f"splice_{i}"] = out.numpy()
        d[f"splice_{i}_got_input_ids"] = np.bool_(seen["input_ids"] is not None)
    for i, (drop_prob, n_dm) in enumerate(PS.CAUSAL_CASES):
        r = PS.live_causal(drop_prob, n_dm)
        d[f"causal_{i}_enc"] = r["enc"].numpy()
        d[f"causal_{i}_lm_loss"] = np.float64(float(r["lm_loss"]))
        d[f"causal_{i}_loss"] = np.float64(float(r["loss"]))
        d[f"causal_{i}_n_model_calls"] = np.int64(r["n_model_calls"])
        if r["u_enc"] is not None:
            d[f"causal_{i}_u_enc"] = r["u_enc"].numpy()
            d[f"causal_{i}_null_ids"] = np.asarray(r["null_ids"])
    for i, case in enumerate(PS.SDHEAD_CASES):
        d[f"sdhead_{i}"] = np.float64(float(PS.live_sdhead(*case)))
    head, _, _, _ = PS.live_sdhead_object(0.0, 0.0, None, None)      # images=None branch (:500-509): DDP's unused-parameter pass
    d["sdhead_dummy"] = np.float64(float(head.forward(None, None, None, dream_embeddings=torch.randn(1, 5, 40))))
    np.savez_compressed(OUT, **d)
    print(f"wrote {OUT}: {len(d)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
