"""TEST INFRASTRUCTURE — golden fixture of LSeg's normalised pixel embedding (image_features) from the REAL reference.

Needs a lang-seg checkout named by LSEG_REFERENCE_ROOT: builds the unmodified reference LSegNet (oracle/ref_standins.py)
on the seeded synthetic state dict (oracle/synth.py), hooks scratch.head1, normalises its output the way
modules/models/lseg_net.py:187-191 does (NHWC rows / their L2 norm), checks that the oracle restatement
(oracle/embed_oracle.py on oracle/lseg_oracle.py's path_1) reproduces it, and writes tests/golden/ref_embed.npz (fp32
NCHW, ~0.6 MB):

  small       B=2, 64x96 (the images of ref_small.npz): an 8x12 lattice (stride 4) of the 32x48 grid, all 512 channels
  s480        B=1, 480x480 (the image of ref_480_k150.npz): a 10x10 lattice (stride 24) of the 240x240 grid, all channels

Usage:  LSEG_REFERENCE_ROOT=/path/to/lang-seg python oracle/make_golden_embed.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import embed_oracle as E  # noqa: E402
from oracle import lseg_oracle as O  # noqa: E402
from oracle import ref_standins as R  # noqa: E402
from oracle import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
CASES = {"small": dict(B=2, H=64, W=96, seed=2064, stride=4), "s480": dict(B=1, H=480, W=480, seed=1480, stride=24)}


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    sd = synth.make_state_dict(0)
    labels = synth.ade20k_labels()[:5]
    net = R.build_reference_net(sd, labels)
    cap = {}
    net.scratch.head1.register_forward_hook(lambda m, a, o: cap.__setitem__("head1", o.detach()))
    out = {}
    for tag, c in CASES.items():
        x = synth.make_image(c["B"], c["H"], c["W"], seed=c["seed"])
        with torch.no_grad():
            net(x)
        f = cap["head1"]
        imshape = f.shape
        rows = f.permute(0, 2, 3, 1).reshape(-1, imshape[1])
        rows = rows / rows.norm(dim=-1, keepdim=True)
        ref = rows.view(imshape[0], imshape[2], imshape[3], imshape[1]).permute(0, 3, 1, 2)
        _, st = O.lseg_forward(x, synth.tokenize(labels), sd, return_stages=True)
        err = ((ref - E.image_features(st["path_1"], sd)).abs().max() / ref.abs().max()).item()
        print(f"{tag}: oracle image_features vs reference max rel err {err:.3e}")
        assert err <= 1e-5, (tag, err)
        s = c["stride"]
        out[tag] = ref[:, :, ::s, ::s].contiguous().numpy().astype(np.float32)
        out[f"{tag}_stride"] = np.array(s)
    np.savez_compressed(os.path.join(GOLD, "ref_embed.npz"), **out)
    print("written", os.path.join(GOLD, "ref_embed.npz"), {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
