"""Writes tests/golden/reference_outputs.npz FROM THE REFERENCE ITSELF (oracle/_ref: GSLAM's own SE3, layouts and Vocabulary,
compiled from the reference headers): what tests/test_oracle_ba.py, test_oracle_posegraph.py and test_oracle_bow.py compare the
oracle against where oracle/_ref is not built.  Exact outputs of the vocabulary are stored as digests (oracle.digest).
Run:  GSLAM_REFERENCE=<GSLAM checkout> python tests/golden/make_golden_reference.py"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from oracle import oracle as O  # noqa: E402
from gslam_b200 import synth  # noqa: E402

LAYOUT = ("KeyPoint", "SE3", "SIM3", "Point3d", "BundleEdge", "KeyFrameEstimzation", "MapPointEstimation", "GImage")
KEYS = ("words", "values", "fv_node", "fv_feat")
N_SE3 = 64


def rand_pose(rng):
    q = rng.standard_normal(4); q /= np.linalg.norm(q)
    return np.concatenate([q, rng.standard_normal(3)])


def queries(v, n, seed, flip=0.05):
    rng = np.random.default_rng(seed)
    src = v.desc[rng.integers(1, v.n_nodes, n)]
    return src ^ np.packbits(rng.random((n, 256)) < flip, axis=1)


def main():
    oracle.build()
    assert oracle.have_ref(), "oracle/_ref is not built: set GSLAM_REFERENCE to a GSLAM checkout"
    R = oracle.ref()
    out = {"layout_names": np.array(LAYOUT), "layout_sizes": np.array([R.ref_sizeof(k.encode()) for k in LAYOUT], np.int32)}
    offs = (C.c_int * 7)(); R.ref_keypoint_offsets(offs); out["kp_offsets"] = np.array(list(offs), np.int32)
    p = rand_pose(np.random.default_rng(0)); raw = np.zeros(8); R.ref_sim3_raw(p.ctypes.data, 2.5, raw.ctypes.data)
    out["sim3_pose"], out["sim3_raw"] = p, raw
    # SE3: inverse, transform, exp * T (test_oracle_ba.test_se3_conventions_match_reference)
    rng = np.random.default_rng(1)
    T, P, D, INV, Q, EXPMUL = [], [], [], [], [], []
    for _ in range(N_SE3):
        t = rand_pose(rng); pt = rng.standard_normal(3); d = 0.3 * rng.standard_normal(6)
        inv = np.zeros(7); R.ref_se3_inverse(t.ctypes.data, inv.ctypes.data)
        q = np.zeros(3); R.ref_se3_transform(inv.ctypes.data, pt.ctypes.data, q.ctypes.data)
        e = np.zeros(7); R.ref_se3_exp(d.ctypes.data, e.ctypes.data)
        w = np.zeros(7); R.ref_se3_mul(e.ctypes.data, t.ctypes.data, w.ctypes.data)
        T.append(t); P.append(pt); D.append(d); INV.append(inv); Q.append(q); EXPMUL.append(w)
    out.update(se3_T=np.array(T), se3_p=np.array(P), se3_d=np.array(D), se3_inv=np.array(INV), se3_q=np.array(Q), se3_expmul=np.array(EXPMUL))
    # SE3 log and product (test_oracle_posegraph.test_se3_log_and_product_equal_the_reference_class)
    rng = np.random.default_rng(0)
    A, B, LOG, MUL = [], [], [], []
    for k in range(N_SE3):
        scale = [1e-12, 1e-6, 0.3, 2.5][k % 4]
        a = synth._small_se3(rng, 1, 1.0, scale)[0]; b = synth._small_se3(rng, 1, 2.0, 1.0)[0]
        if k % 7 == 0:
            a[:4] = -a[:4]
        lg = np.zeros(6); R.ref_se3_log(a.ctypes.data, lg.ctypes.data)
        m = np.zeros(7); R.ref_se3_mul(a.ctypes.data, b.ctypes.data, m.ctypes.data)
        A.append(a); B.append(b); LOG.append(lg); MUL.append(m)
    out.update(pg_a=np.array(A), pg_b=np.array(B), pg_log=np.array(LOG), pg_mul=np.array(MUL))
    dig = {}
    # Vocabulary::transform, every weighting and scoring (test_oracle_bow.test_every_weighting_and_scoring_against_live_reference)
    for weighting in (O.W_TF_IDF, O.W_TF, O.W_IDF, O.W_BINARY):
        for scoring in (O.S_L1, O.S_L2, O.S_CHI_SQUARE, O.S_KL, O.S_BHATTACHARYYA, O.S_DOT_PRODUCT):
            v = O.synth_vocabulary(10, 3, seed=7, weighting=weighting, scoring=scoring, stop=0.1)
            rv = O.RefVocabulary.from_arrays(v)
            f = queries(v, 700, seed=weighting * 10 + scoring)
            for lu in (0, 1, 3, 5):
                want = rv.transform(f, lu)
                for k in KEYS:
                    dig[f"bow_w{weighting}_s{scoring}_lu{lu}_{k}"] = oracle.digest(want[k])
            rv.close()
    # a tree trained by Vocabulary::create (test_trained_vocabulary_against_live_reference)
    rng = np.random.default_rng(5)
    centres = rng.integers(0, 256, (300, 32), dtype=np.uint8)
    train = centres[rng.integers(0, 300, (40, 200))] ^ np.packbits(rng.random((40, 200, 256)) < 0.06, axis=2)
    rv = O.RefVocabulary.train(train, 40, 10, 3)
    v = rv.arrays()
    out.update(trained_kLws=np.array([v.k, v.L, v.weighting, v.scoring], np.int32), trained_child_num=v.child_num, trained_weight=v.weight,
               trained_desc=v.desc)
    f = queries(v, 1000, seed=1)
    for lu in (0, 1, 2):
        want = rv.transform(f, lu)
        for k in KEYS:
            dig[f"trained_lu{lu}_{k}"] = oracle.digest(want[k])
    one = [rv.transform_one(f[i], 1) for i in range(0, 1000, 97)]
    out["trained_one_word_node"] = np.array([(w, n) for w, _, n in one], np.int64)
    rv.close()
    # a pruned tree with ten-way ties (test_unbalanced_tree_and_ties)
    v = O.synth_vocabulary(10, 4, seed=3, prune=0.15, stop=0.05)
    v.desc[11:21] = v.desc[11]
    rv = O.RefVocabulary.from_arrays(v)
    f = queries(v, 1500, seed=9)
    for lu in (0, 4):
        want = rv.transform(f, lu)
        for k in KEYS:
            dig[f"unbalanced_lu{lu}_{k}"] = oracle.digest(want[k])
    rv.close()
    out["digest_names"] = np.array(list(dig)); out["digests"] = np.array(list(dig.values()), "S32")
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_outputs.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
