"""Generates tests/golden/bow_golden.npz FROM THE REFERENCE ITSELF (oracle/_ref = GSLAM::Vocabulary compiled from the reference
headers; needs GSLAM_REFERENCE at build time): a vocabulary trained by Vocabulary::create (k = 8, L = 3, TF_IDF / L1_NORM) on 60
"images" of 150 clustered 256-bit descriptors, exported as flat arrays, plus the BowVector / FeatureVector the reference's
Vocabulary::transform (Vocabulary.h:1558-1622) returns for two query sets at levelsup 0 and 2.

    python tests/golden/make_golden_bow.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import oracle as O  # noqa: E402


def clustered(rng, n_images, per_image, n_centres=200, flip=0.08):
    centres = rng.integers(0, 256, (n_centres, 32), dtype=np.uint8)
    which = rng.integers(0, n_centres, (n_images, per_image))
    noise = np.packbits(rng.random((n_images, per_image, 256)) < flip, axis=2)
    return centres[which] ^ noise


def main():
    rng = np.random.default_rng(2024)
    train = clustered(rng, 60, 150)
    R = O.RefVocabulary.train(train, 60, 8, 3, O.W_TF_IDF, O.S_L1)
    v = R.arrays()
    out = dict(k=v.k, L=v.L, weighting=v.weighting, scoring=v.scoring, child_num=v.child_num, weight=v.weight, desc=v.desc)
    for name, q in (("a", clustered(rng, 1, 500)[0]), ("b", rng.integers(0, 256, (300, 32), dtype=np.uint8))):
        out[f"q_{name}"] = q
        for lu in (0, 2):
            r = R.transform(q, lu)
            for key in ("words", "values", "fv_node", "fv_feat"):
                out[f"{name}_lu{lu}_{key}"] = r[key]
    R.close()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bow_golden.npz")
    np.savez_compressed(path, **out)
    print(path, v.n_nodes, "nodes", int((v.child_num == 0).sum()), "leaves")


if __name__ == "__main__":
    main()
