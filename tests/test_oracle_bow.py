"""Bag-of-words transform (SURVEY.md section 8f-4, GSLAM/core/Vocabulary.h:1558-1736): the oracle's restatement (oracle/bow_ref.c)
against golden vectors produced by the reference itself (tests/golden/make_golden_bow.py) and, where oracle/_ref is built, against
the live reference -- Vocabulary::create-trained and Vocabulary::load-ed trees, every weighting and scoring type."""
import os

import numpy as np
import pytest

import oracle
from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bow_golden.npz")
KEYS = ("words", "values", "fv_node", "fv_feat")
# the reference's outputs (tests/golden/make_golden_reference.py): exact results as digests, the trained tree as arrays
_Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs.npz"))
STORED = {**{k: _Z[k] for k in _Z.files if k.startswith("trained_")}, **dict(zip(_Z["digest_names"].tolist(), _Z["digests"].tolist()))}


def golden_vocabulary():
    z = np.load(GOLD)
    return z, O.VocabularyArrays(int(z["k"]), int(z["L"]), int(z["weighting"]), int(z["scoring"]), z["child_num"], z["weight"], z["desc"])


def queries(v, n, seed, flip=0.05):
    """descriptors a few bit flips away from random nodes of the tree (so that the walk is decided by small distances, ties included)"""
    rng = np.random.default_rng(seed)
    src = v.desc[rng.integers(1, v.n_nodes, n)]
    return src ^ np.packbits(rng.random((n, 256)) < flip, axis=1)


@pytest.mark.parametrize("q", ["a", "b"])
@pytest.mark.parametrize("lu", [0, 2])
def test_oracle_equals_reference_golden(q, lu):
    z, v = golden_vocabulary()
    got = O.bow_transform(v, z[f"q_{q}"], lu)
    for k in KEYS:
        assert np.array_equal(got[k], z[f"{q}_lu{lu}_{k}"]), k
    assert abs(float(got["values"].sum()) - 1.0) < 1e-5    # L1-normalised
    assert np.all(np.diff(got["words"]) > 0)               # std::map order


def test_golden_vocabulary_is_a_trained_tree():
    z, v = golden_vocabulary()
    assert v.k == 8 and v.L == 3 and v.n_nodes == (8 ** 4 - 1) // 7
    leaves = v.child_num == 0
    assert leaves.sum() > 100 and np.all(v.weight[leaves] >= 0)
    # the export is loadable by the reference's own binary loader and walks identically
    if oracle.have_ref():
        R = O.RefVocabulary.from_arrays(v)
        r = R.transform(z["q_a"], 1)
        g = O.bow_transform(v, z["q_a"], 1)
        assert all(np.array_equal(g[k], r[k]) for k in KEYS)
        R.close()


def _stored(name):
    return STORED[name].decode()


def _reference_vs_stored(R, f, lu, prefix):
    """The live reference's transform (oracle/_ref) must still give the stored digests."""
    want = R.transform(f, lu)
    for k in KEYS:
        assert oracle.digest(want[k]) == _stored(f"{prefix}_{k}"), (prefix, k)


@pytest.mark.parametrize("weighting", [O.W_TF_IDF, O.W_TF, O.W_IDF, O.W_BINARY])
@pytest.mark.parametrize("scoring", [O.S_L1, O.S_L2, O.S_CHI_SQUARE, O.S_KL, O.S_BHATTACHARYYA, O.S_DOT_PRODUCT])
def test_every_weighting_and_scoring_against_live_reference(weighting, scoring):
    """Against Vocabulary::transform: live where oracle/_ref is built, and always against its outputs stored as digests in
    tests/golden/reference_outputs.npz."""
    v = O.synth_vocabulary(10, 3, seed=7, weighting=weighting, scoring=scoring, stop=0.1)
    f = queries(v, 700, seed=weighting * 10 + scoring)
    R = O.RefVocabulary.from_arrays(v) if oracle.have_ref() else None
    for lu in (0, 1, 3, 5):
        prefix = f"bow_w{weighting}_s{scoring}_lu{lu}"
        got = O.bow_transform(v, f, lu)
        for k in KEYS:
            assert oracle.digest(got[k]) == _stored(f"{prefix}_{k}"), (k, lu)
        if R is not None:
            _reference_vs_stored(R, f, lu, prefix)
    if R is not None:
        R.close()


def test_trained_vocabulary_against_live_reference():
    """A tree trained by Vocabulary::create, walked by the oracle and by the reference: the tree and the reference's walks as stored
    in tests/golden/reference_outputs.npz, and a freshly trained tree live where oracle/_ref is built (training leaves some
    weights uninitialised, so a fresh tree is compared with its own live walks only)."""
    kLws = STORED["trained_kLws"]
    stored = O.VocabularyArrays(int(kLws[0]), int(kLws[1]), int(kLws[2]), int(kLws[3]), STORED["trained_child_num"],
                                STORED["trained_weight"], STORED["trained_desc"])
    assert stored.n_nodes == 1111
    f = queries(stored, 1000, seed=1)
    for lu in (0, 1, 2):
        got = O.bow_transform(stored, f, lu)
        for k in KEYS:
            assert oracle.digest(got[k]) == _stored(f"trained_lu{lu}_{k}"), (k, lu)
    got = O.bow_transform(stored, f, 1)
    for j, i in enumerate(range(0, 1000, 97)):   # the single-descriptor walk
        want = tuple(int(x) for x in STORED["trained_one_word_node"][j])
        assert want == (int(got["f_word"][i]), int(O.bow_transform(stored, f[i:i + 1], 1)["f_node"][0]))
    if not oracle.have_ref():
        return
    rng = np.random.default_rng(5)
    centres = rng.integers(0, 256, (300, 32), dtype=np.uint8)
    train = centres[rng.integers(0, 300, (40, 200))] ^ np.packbits(rng.random((40, 200, 256)) < 0.06, axis=2)
    R = O.RefVocabulary.train(train, 40, 10, 3)
    v = R.arrays()
    assert v.n_nodes == 1111
    f = queries(v, 1000, seed=1)
    for lu in (0, 1, 2):
        want = R.transform(f, lu); got = O.bow_transform(v, f, lu)
        for k in KEYS:
            assert np.array_equal(got[k], want[k]), (k, lu)
    for i in range(0, 1000, 97):
        w, val, node = R.transform_one(f[i], 1)
        assert (w, node) == (int(got["f_word"][i]), int(O.bow_transform(v, f[i:i + 1], 1)["f_node"][0]))
    R.close()


def test_unbalanced_tree_and_ties():
    """Pruned trees (leaves above level L, inner nodes with fewer than k children) and exact distance ties (first child wins)."""
    v = O.synth_vocabulary(10, 4, seed=3, prune=0.15, stop=0.05)
    v.desc[11:21] = v.desc[11]           # the ten children of node 1 are identical: every query reaching node 1 ties ten ways
    f = queries(v, 1500, seed=9)
    R = O.RefVocabulary.from_arrays(v) if oracle.have_ref() else None
    got = O.bow_transform(v, f, 0)
    assert oracle.digest(got["words"]) == _stored("unbalanced_lu0_words") and oracle.digest(got["values"]) == _stored("unbalanced_lu0_values")
    under1 = got["f_word"][(got["f_word"] >= 11) & (got["f_word"] <= 20)]
    assert under1.size == 0 or np.all(under1 == 11)
    # levelsup >= L: every feature files under the root (Vocabulary.h:1699-1700)
    top = O.bow_transform(v, f, 4)
    assert np.all(top["fv_node"] == 0)
    assert oracle.digest(top["fv_node"]) == _stored("unbalanced_lu4_fv_node") and oracle.digest(top["fv_feat"]) == _stored("unbalanced_lu4_fv_feat")
    if R is not None:
        _reference_vs_stored(R, f, 0, "unbalanced_lu0")
        _reference_vs_stored(R, f, 4, "unbalanced_lu4")
        R.close()
    # our definition where the reference reads an uninitialised nid: a leaf above the requested level files under itself
    shallow = v.child_num[got["f_word"]] == 0
    assert shallow.all()
    early = got["f_word"] < (10 ** 4 - 1) // 9    # leaves above level 4
    assert early.any() and np.array_equal(got["f_node"][early], got["f_word"][early])


def test_empty_and_single_inputs():
    z, v = golden_vocabulary()
    e = O.bow_transform(v, np.zeros((0, 32), np.uint8), 0)
    assert all(e[k].size == 0 for k in KEYS)
    one = O.bow_transform(v, z["q_a"][:1], 0)
    assert one["words"].size == 1 and one["values"][0] == np.float32(1.0) and one["fv_feat"].tolist() == [0]


# ---- the cases of tests/_bow_cases.py: boundaries of the device's launch plan, and the norm's order of summation ------------------
import _bow_cases as BC  # noqa: E402


@pytest.mark.parametrize("case", BC.CASES, ids=lambda c: c.id)
def test_case_reaches_its_boundary(case):
    """The mirror of the launch plan reaches the boundary each case was written for, and the mirror of the reduce kernel's
    BowVector (words, run sums, norm fold with its exactness predicate) gives the oracle's words and values."""
    BC.check_reach(case)
    v, f, lu = case.data
    ref = O.bow_transform(v, f, lu)
    fold = BC.norm_fold(v, ref)
    assert np.array_equal(fold["words"], ref["words"])
    assert np.array_equal(BC.mirror_values(v, fold), ref["values"])


def test_tree_norm_differs_from_the_reference_on_the_adversarial_case():
    """IDF / L1 over 65 538 words (1, w, and 65 536 x 2^-54): the norm folded in the kernel's tree keeps 2^-38 that the reference's
    sequential sum absorbs, and the second word's value comes out one float apart -- unless the sequential re-sum runs."""
    v, f, lu = BC.BY_ID["norm_adversarial"].data
    ref = O.bow_transform(v, f, lu)
    fold = BC.norm_fold(v, ref)
    assert fold["tree"] != fold["seq"] and fold["q"] == -54 and BC.sequential_needed(fold)
    tree = BC.normalise(v, fold, fold["tree"])
    diff = np.nonzero(tree != ref["values"])[0]
    assert diff.tolist() == [1] and ref["values"][1] == np.float32(0.26592186) and tree[1] == np.float32(0.26592183)
    assert np.array_equal(BC.normalise(v, fold, fold["seq"]), ref["values"])


@pytest.mark.parametrize("cid", ["norm_inside_l1", "norm_inside_l2", "norm_l1_bench_like", "norm_l2_bench_like", "norm_l1_wide_idf"])
def test_tree_norm_equals_the_reference_inside_the_bound(cid):
    v, f, lu = BC.BY_ID[cid].data
    ref = O.bow_transform(v, f, lu)
    fold = BC.norm_fold(v, ref)
    assert not BC.sequential_needed(fold)
    assert fold["tree"] == fold["seq"] and np.array_equal(BC.normalise(v, fold, fold["tree"]), ref["values"])


def test_plan_mirror_at_device_counts():
    """npad is launched for the capacity and clipped to the count's power of two (at least 2) on the device."""
    assert BC.plan(10, 3000, 0) == (16, 1, 4096, 2, 1)
    assert BC.plan(10, 3000, 1) == (16, 1, 4096, 2, 1)
    assert BC.plan(20, 3000, 1234) == (32, 1, 4096, 2048, 2)
    assert BC.plan(10, 12000, 8192) == (16, 0, 16384, 8192, 8)
    assert BC.plan(10, 12000, 8193) == (16, 0, 16384, 16384, 16)
    assert BC.plan(10, 12000, 12000) == (16, 0, 16384, 16384, 16)
    assert BC.plan(17, 1, None) == (32, 1, 2, 2, 1) and BC.plan(16, 0, None) == (0, 0, 0, 0, 0)


@pytest.mark.parametrize("case", BC.CASES, ids=lambda c: c.id)
def test_case_oracle_equals_live_reference(case):
    """Where oracle/_ref is built: the oracle equals Vocabulary::transform on every case the reference defines (not a negative
    levelsup, no walk ending above level L - levelsup: the reference reads an uninitialised node id there)."""
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built")
    if not BC.reference_defined(case):
        pytest.skip("the reference leaves the node id undefined here")
    v, f, lu = case.data
    R = O.RefVocabulary.from_arrays(v)
    try:
        want = R.transform(f, lu)
    finally:
        R.close()
    got = O.bow_transform(v, f, lu)
    for k in KEYS:
        assert np.array_equal(got[k], want[k], equal_nan=k == "values"), k
