"""Golden fixture for the 3-D centre parse on a volume with far more local maxima than 64 (and than 4096): the
REFERENCE's own CenterMap3D.parse_3dcentermap (bev/post_parser.py:44-66) on synth.bev_noise_volume (build container
only).    python tests/golden/make_golden_bev_parse_dense.py"""
import importlib
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
from make_golden import load_reference  # noqa: E402

SEED, THRESH = 20, 0.08


def main():
    from romp_b200 import synth
    load_reference()
    PP = importlib.import_module("bev.post_parser")
    vol = torch.from_numpy(synth.bev_noise_volume(SEED))
    with torch.no_grad():
        bi, czyx, conf = PP.CenterMap3D(THRESH).parse_3dcentermap(vol)
        nm = vol * (F.max_pool3d(vol, 5, 1, 2) == vol).float()
    s = torch.sort(nm.reshape(-1), descending=True).values
    n_max = int((s > THRESH).sum())
    # the top-64 is defined without a tie rule: 64 distinct scores, strictly above the 65th
    assert len(bi) == 64 and len(set(conf.tolist())) == 64 and s[63] > s[64] and n_max > 4096
    np.savez_compressed(os.path.join(HERE, "bev_parse_dense.npz"), seed=SEED, thresh=THRESH, n_maxima=n_max,
                        batch_ids=bi.numpy(), czyx=czyx.numpy(), conf=conf.numpy())
    print("bev_parse_dense.npz:", n_max, "local maxima above", THRESH)


if __name__ == "__main__":
    main()
