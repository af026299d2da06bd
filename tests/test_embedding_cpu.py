"""CPU: the oracle's normalised pixel embedding (`image_features`, lseg_net.py:185-191) against the output of the
unmodified reference (tests/golden/ref_embed.npz, oracle/make_golden_embed.py). The image path is restated op for op, so
the two agree at the fp32 level the other oracle fixtures are held to."""
import os

import numpy as np
import pytest
import torch

from oracle import embed_oracle as E
from parity_util import O, state_dict, synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
FP32_TOL = 1e-6  # max |oracle - reference| on unit-norm rows: a few fp32 ulps of the largest component


@pytest.mark.parametrize("tag,B,H,W,seed", [("small", 2, 64, 96, 2064), ("s480", 1, 480, 480, 1480)])
def test_image_features_match_reference(tag, B, H, W, seed):
    z = np.load(os.path.join(GOLD, "ref_embed.npz"))
    s = int(z[f"{tag}_stride"])
    x = synth.make_image(B, H, W, seed=seed)
    _, st = O.lseg_forward(x, synth.tokenize(["cat", "other"]), state_dict(0), return_stages=True)
    f = E.image_features(st["path_1"], state_dict(0))
    assert f.shape == (B, 512, H // 2, W // 2) and f.dtype == torch.float32
    ref = torch.from_numpy(z[tag])
    got = f[:, :, ::s, ::s]
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= FP32_TOL
    norms = f.norm(dim=1)
    assert (norms - 1).abs().max().item() < 1e-5  # unit rows, as the reference normalises them
