"""TEST INFRASTRUCTURE — golden fixture of the ViT's recorded attention maps from the REAL reference.

Needs a lang-seg checkout named by LSEG_REFERENCE_ROOT. Builds the unmodified reference LSegNet (oracle/ref_standins.py)
on the seeded synthetic state dict (oracle/synth.py), then swaps in the encoder that the reference's own
_make_encoder(..., enable_attention_hooks=True) builds (modules/models/lseg_blocks.py:12-57; LSeg.__init__ never forwards
the flag, lseg_net.py:126-134), reloads the state dict, runs the net and reads pretrained.attention — the reference's
hooks (get_attention, lseg_vit.py:22-42), not a restatement. Checks that oracle/vit_attention_oracle.py reproduces it and
writes tests/golden/ref_attention.npz (fp32):

  small_attn_1..4      B=2, 64x96 (N = 25): the full [2, 16, 25, 25] tensors
  s480_attn_1..4       B=1, 480x480 (N = 901): rows s480_rows = {0, 465} of every head, [1, 16, 2, 901]
  mean_b1_t<token>_attn_k  the reference's get_mean_attention_map(attn_k[:1], token, (1, 3, 64, 96)), [64, 96], for
                           tokens 0 and 7 of attn_1 and attn_4
  mean_b2_t<token>_attn_k  the same on both images (its B > 1 behaviour: the mean runs over the images, leaving
                           [16, 64, 96]), stored on the pixel lattice [:, ::8, ::8] to keep the file under 1 MB

Usage:  LSEG_REFERENCE_ROOT=/path/to/lang-seg python oracle/make_golden_attention.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_standins as R  # noqa: E402
from oracle import synth  # noqa: E402
from oracle import vit_attention_oracle as A  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
CASES = {"small": dict(B=2, H=64, W=96, seed=2064), "s480": dict(B=1, H=480, W=480, seed=1480)}
S480_ROWS = (0, 465)
MEAN_TOKENS = (0, 7)
MEAN_BLOCKS = ("attn_1", "attn_4")
MEAN_B2_STRIDE = 8


def reference_with_attention_hooks(sd, labels):
    """The reference net whose encoder was built with enable_attention_hooks=True, weights loaded."""
    net = R.build_reference_net(sd, labels)
    cwd = os.getcwd()
    os.chdir(R.REFERENCE_ROOT)
    try:
        from modules.models.lseg_blocks import _make_encoder
        _, pretrained, _ = _make_encoder("clip_vitl16_384", 256, groups=1, expand=False, exportable=False,
                                         hooks=[5, 11, 17, 23], use_readout="project", enable_attention_hooks=True)
    finally:
        os.chdir(cwd)
    net.pretrained = pretrained
    missing, unexpected = net.load_state_dict(sd, strict=False)
    missing = [k for k in missing if "num_batches_tracked" not in k]
    assert not missing, missing[:5]
    assert hasattr(net.pretrained, "attention")
    return net.eval()


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    sd = synth.make_state_dict(0)
    labels = synth.ade20k_labels()[:5]
    net = reference_with_attention_hooks(sd, labels)
    from modules.models.lseg_vit import get_mean_attention_map
    out = {}
    for tag, c in CASES.items():
        x = synth.make_image(c["B"], c["H"], c["W"], seed=c["seed"])
        with torch.no_grad():
            net(x)
        ref = {k: v.detach().clone() for k, v in net.pretrained.attention.items()}
        assert sorted(ref) == ["attn_1", "attn_2", "attn_3", "attn_4"], sorted(ref)
        ours = A.vit_attention_maps(x, sd)
        for k in ref:
            err = (ref[k] - ours[k]).abs().max().item()
            print(f"{tag} {k}: oracle vs reference max abs err {err:.3e}")
            assert err <= 1e-6, (tag, k, err)
            if tag == "small":
                out[f"small_{k}"] = ref[k].numpy().astype(np.float32)
            else:
                out[f"s480_{k}"] = ref[k][:, :, list(S480_ROWS)].contiguous().numpy().astype(np.float32)
        if tag == "small":
            shape1, shape2 = (1, 3, c["H"], c["W"]), (2, 3, c["H"], c["W"])
            for k in MEAN_BLOCKS:
                for t in MEAN_TOKENS:
                    out[f"mean_b1_t{t}_{k}"] = get_mean_attention_map(ref[k][:1], t, shape1).numpy().astype(np.float32)
                    m2 = get_mean_attention_map(ref[k], t, shape2)
                    assert m2.shape == (16, c["H"], c["W"]), m2.shape
                    s2 = MEAN_B2_STRIDE
                    out[f"mean_b2_t{t}_{k}"] = m2[:, ::s2, ::s2].contiguous().numpy().astype(np.float32)
    out["s480_rows"] = np.array(S480_ROWS)
    out["mean_tokens"] = np.array(MEAN_TOKENS)
    out["mean_b2_stride"] = np.array(MEAN_B2_STRIDE)
    path = os.path.join(GOLD, "ref_attention.npz")
    np.savez_compressed(path, **out)
    print("written", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
