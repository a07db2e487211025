"""Bag-of-words transform cases at the boundaries of its launch plan, shared by the CPU checks of the plan and of the norm
(tests/test_oracle_bow.py) and the device-vs-oracle parity tests (tests/test_bow_paths_gpu.py).

gb_bow_transform (gslam_b200/csrc/bow.cu) walks each descriptor down the tree with a group of G lanes (16 when k <= 16, else 32;
lane c reads child c), then one 1024-thread CTA sorts (word, feature) and (node, feature) keys: npad = the power of two >= n (at
least 2) keys, in shared memory up to 8192 and in global memory above.  While the row count is still on the device the launch
covers the capacity and the kernel clips npad to the count's power of two.  Every thread reads a chunk of per = npad / 1024 sorted
keys; a word's run of equal keys is summed by the thread holding its first key, past its chunk if the run goes on.  The node keys
are sorted only when some live feature's node differs from its word (`same`).  The double L1 / L2 norm is folded in a fixed tree
(thread chunks, warp shuffles, a tree over the warps); when that total is not below 2^(q+52), q the smallest exponent of the
lowest set bit of a term, one thread re-sums it in word order.

`plan` and `norm_fold` mirror all of that; each case states the boundary it exists to reach as facts, which `check_reach`
asserts, so that an edit to a case or to the kernel's plan cannot quietly turn a boundary case into an easy one.

Facts:
  G, in_smem, npad, npad_sorted, per     the plan's value
  same / sequential                      the node sort is skipped / the norm is re-summed in word order
  k, n, root_only, deeper_than_L, leaves_level1, nodes_min   the tree and the row count
  hits_child_ge16                        some walk takes child 16 or later (missed by a 16-lane walk)
  fewer_children                         some walk passes an inner node with fewer than k children
  lu                                     levelsup relative to L: "neg", "0", "1", "L-1", "L", "L+3"
  ng_mod256                              n * G is not a multiple of 256 (a partial walk CTA)
  run_starts_chunk / run_ends_chunk      some run of a word starts on a chunk's first key / ends on a chunk's last key
  run_spans                              some run covers at least this many chunks
  run_all                                one word is hit by every row
  one_differ                             exactly one live feature's node differs from its word, its index not a multiple of 1024,
                                         its word key in the last chunk that holds keys
  differ_stopped                         a feature whose node differs from its word is stopped (and `same` holds)
  nw                                     the number of words
  weights                                kinds of weight on words the walks hit: "neg_zero", "negative", "nan", "subnormal"
  tree_differs                           the tree-folded norm gives other values than the reference's order
  bound_inside                           the tree total lies in [2^(q+51), 2^(q+52)): exact, and within a factor 2 of the bound
"""
import dataclasses
import functools
import math

import numpy as np

from oracle import oracle as O

SMEM_KEYS = 8192
RED_THREADS = 1024
WALK_THREADS = 256
TF_WEIGHTINGS = (O.W_TF, O.W_TF_IDF)


def next_pow2(n):
    p = 2
    while p < n:
        p <<= 1
    return p


def plan(k, n, count=None):
    """Mirror of bow_run's launch and of the reduce kernel's clip -> (G, in_smem, npad launched, npad sorted, per).  n: the rows
    launched (the capacity while the count is on the device), count: the device-side count or None.  All 0: no launch."""
    if n == 0:
        return 0, 0, 0, 0, 0
    g = 16 if k <= 16 else 32
    npad = next_pow2(n)
    sorted_ = npad if count is None else min(npad, next_pow2(max(0, min(n, count))))
    return g, int(npad <= SMEM_KEYS), npad, sorted_, (sorted_ + RED_THREADS - 1) // RED_THREADS


def lsb_exponent(t):
    """t >= 0, a float32: the exponent q of its lowest set bit (t = odd * 2^q); None for 0."""
    b = int(np.float32(t).view(np.uint32))
    if b == 0:
        return None
    e, m = b >> 23, b & 0x7FFFFF
    sig = (m | 0x800000) if e else m
    return (e - 150 if e else -149) + ((sig & -sig).bit_length() - 1)


def _tree32(a):
    """lane 0 of `v += __shfl_down_sync(v, o)` for o = 16 .. 1 (a lane past the warp reads its own value)"""
    a = list(a)
    for o in (16, 8, 4, 2, 1):
        a = [a[l] + (a[l + o] if l + o < 32 else a[l]) for l in range(32)]
    return a[0]


def live_keys(voc, ref, count=None):
    """(word, feature) of the live features in sorted key order, as the reduce kernel holds them; `ref`: oracle.bow_transform of
    the rows launched."""
    fw = ref["f_word"]
    n = len(fw) if count is None else min(len(fw), count)
    w = voc.weight[fw[:n]]
    with np.errstate(invalid="ignore"):
        live = np.nonzero(w > 0)[0]
    order = np.lexsort((live, fw[live]))
    return fw[live][order], live[order]


def norm_fold(voc, ref, count=None, per=None):
    """Mirror of the reduce kernel's BowVector and norm: -> dict(words, raw (float32 values before normalisation), terms, tree,
    seq (the reference's sum in word order), q, heads (sorted position of each word's first key), per)."""
    kw, _ = live_keys(voc, ref, count)
    m = len(kw)
    if per is None:
        n = len(ref["f_word"]) if count is None else count
        per = plan(voc.k, max(n, 1), None)[4]
    tf = voc.weighting in TF_WEIGHTINGS
    heads = [i for i in range(m) if i == 0 or kw[i - 1] != kw[i]]
    ends = heads[1:] + [m]
    raw, terms = [], []
    for h, e in zip(heads, ends):
        w = np.float32(voc.weight[kw[h]])
        v = w
        if tf:
            for _ in range(e - h - 1):
                v = np.float32(v + w)
        raw.append(v)
        terms.append(np.float32(v * v) if voc.scoring == O.S_L2 else np.float32(abs(v)))
    local = [0.0] * RED_THREADS
    for h, t in zip(heads, terms):
        local[h // per] += float(t)
    tree = _tree32([_tree32(local[32 * w:32 * w + 32]) for w in range(32)])
    seq = 0.0
    for t in terms:
        seq += float(t)
    qs = [q for q in (lsb_exponent(t) for t in terms) if q is not None]
    return dict(words=np.asarray([kw[h] for h in heads], np.int64), raw=np.asarray(raw, np.float32), terms=terms, tree=tree, seq=seq,
                q=min(qs) if qs else None, heads=heads, ends=ends, per=per)


def sequential_needed(fold):
    """The kernel's predicate: the tree total is not below 2^(q+52)."""
    if fold["q"] is None:
        return not (fold["tree"] < math.inf)
    return not (fold["tree"] < math.ldexp(1.0, fold["q"] + 52))


def normalise(voc, fold, norm):
    """The values as the kernel writes them with the un-rooted norm `norm` (the tree's or the sequential one)."""
    raw = fold["raw"]
    must = voc.scoring != O.S_DOT_PRODUCT
    tf = voc.weighting in TF_WEIGHTINGS
    if not must:
        if not tf or len(raw) == 0:
            return raw.copy()
        norm = float(len(raw))
    elif voc.scoring == O.S_L2:
        norm = math.sqrt(norm)
    if not norm > 0.0:
        return raw.copy()
    return np.asarray([np.float32(float(v) / norm) for v in raw], np.float32)


def mirror_values(voc, fold):
    """The kernel's values, predicate included."""
    must = voc.scoring != O.S_DOT_PRODUCT
    return normalise(voc, fold, fold["seq"] if must and sequential_needed(fold) else fold["tree"])


def flags(voc, ref, fold, count=None):
    """The plan's flags word: 1 = node keys not sorted, 2 = norm re-summed in word order."""
    n = len(ref["f_word"]) if count is None else min(len(ref["f_word"]), count)
    w = voc.weight[ref["f_word"][:n]]
    with np.errstate(invalid="ignore"):
        live = w > 0
    same = bool(np.all(ref["f_word"][:n][live] == ref["f_node"][:n][live]))
    seq = voc.scoring != O.S_DOT_PRODUCT and sequential_needed(fold)
    return (1 if same else 0) | (2 if seq else 0)


def device_plan(voc, ref, n, count=None):
    """The five values gb_dbg_bow_last_plan reports for a launch of n rows (count: the device-side count)."""
    g, sm, npad, npad_sorted, per = plan(voc.k, n, count)
    if g == 0:
        return (0, 0, 0, 0, 0)
    fold = norm_fold(voc, ref, count, per)
    return (g, sm, npad, npad_sorted, flags(voc, ref, fold, count))


# ---- trees ---------------------------------------------------------------------------------------------------------------------
def n_complete(k, L):
    return L + 1 if k == 1 else (k ** (L + 1) - 1) // (k - 1)


def digit_tree(k, L, seed=0, weighting=O.W_TF_IDF, scoring=O.S_L1):
    """A complete k-ary tree of depth L whose node descriptors spell their path: level l owns bits [k*(l-1), k*l), one bit per
    digit.  A query that spells a leaf's path (digit_query) walks to that leaf and nowhere else: at each level the child with the
    query's digit is 2 bits closer than its siblings.  Needs k * L <= 256."""
    assert k * L <= 256
    rng = np.random.default_rng(seed)
    n = n_complete(k, L)
    child = np.zeros(n, np.uint32)
    child[:n_complete(k, L - 1) if L > 0 else 0] = k
    bits = np.zeros((n, 256), np.uint8)
    lo = 1
    for lvl in range(1, L + 1):  # a node's bits: its parent's, and its own digit at its level
        ids = np.arange(lo, n_complete(k, lvl))
        bits[ids] = bits[(ids - 1) // k]
        bits[ids, k * (lvl - 1) + (ids - 1) % k] = 1
        lo = n_complete(k, lvl)
    weight = rng.uniform(0.2, 9.0, n).astype(np.float32)
    return O.VocabularyArrays(k, L, weighting, scoring, child, weight, np.packbits(bits, axis=1))


def depths(k, ids):
    """levels of the nodes `ids` in the implicit k-ary layout (root 0)"""
    ids = np.asarray(ids, np.int64).copy()
    d = np.zeros(ids.shape, np.int64)
    while (ids > 0).any():
        nz = ids > 0
        ids[nz] = (ids[nz] - 1) // k
        d[nz] += 1
    return d


def digit_queries(k, paths):
    """[n][32] descriptors that spell `paths` ([n][depth] digits from the root down)"""
    paths = np.asarray(paths, np.int64).reshape(len(paths), -1)
    bits = np.zeros((len(paths), 256), np.uint8)
    bits[np.arange(len(paths))[:, None], k * np.arange(paths.shape[1])[None, :] + paths] = 1
    return np.packbits(bits, axis=1)


def leaf_paths(k, L, ranks):
    """[n][L] paths of the leaves at level L with ranks `ranks` (0 = the leftmost)"""
    r = np.asarray(ranks, np.int64).copy()
    out = np.zeros((len(r), L), np.int64)
    for lvl in range(L - 1, -1, -1):
        out[:, lvl] = r % k
        r //= k
    return out


def first_leaf(k, L):
    return n_complete(k, L - 1) if L > 0 else 0


def queries(v, n, seed, flip=0.05):
    """descriptors a few bit flips away from random nodes of the tree (ties and near-ties decide many walks)"""
    rng = np.random.default_rng(seed)
    src = v.desc[rng.integers(1, max(v.n_nodes, 2), n) % v.n_nodes]
    return src ^ np.packbits(rng.random((n, 256)) < flip, axis=1)


def with_voc(v, **kw):
    return O.VocabularyArrays(kw.get("k", v.k), kw.get("L", v.L), kw.get("weighting", v.weighting), kw.get("scoring", v.scoring),
                              kw.get("child_num", v.child_num), kw.get("weight", v.weight), kw.get("desc", v.desc))


# ---- cases ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class BowCase:
    id: str
    make: object          # () -> (VocabularyArrays, descriptors [n][32], levelsup)
    reach: tuple = ()

    @functools.cached_property
    def data(self):
        return self.make()


def _c(id, make, **reach):
    return BowCase(id, make, tuple(sorted(reach.items())))


def _walk_width(k, L, n, seed, prune=False):
    def make():
        v = digit_tree(k, L, seed)
        rng = np.random.default_rng(seed)
        if prune:  # inner nodes with fewer than k children, and a few leaves above level L
            inner = n_complete(k, L - 1)
            sel = rng.random(inner) < 0.3
            sel[0] = False
            v.child_num[:inner][sel] = rng.integers(1, k, int(sel.sum()))
            cut = rng.random(inner) < 0.05
            cut[0] = False
            v.child_num[:inner][cut] = 0
        # every digit at every level, then random paths
        paths = np.vstack([(np.arange(k)[:, None] + np.arange(L)[None, :]) % k, rng.integers(0, k, (n - k, L))])
        return v, digit_queries(k, paths), 0
    return make


def _chain(depth, L, n, seed):
    def make():
        rng = np.random.default_rng(seed)
        child = np.ones(depth + 1, np.uint32)
        child[-1] = 0
        weight = rng.uniform(0.2, 9.0, depth + 1).astype(np.float32)
        desc = rng.integers(0, 256, (depth + 1, 32), dtype=np.uint8)
        v = O.VocabularyArrays(1, L, O.W_TF_IDF, O.S_L1, child, weight, desc)
        return v, rng.integers(0, 256, (n, 32), dtype=np.uint8), 1
    return make


def _root_only(n, seed):
    def make():
        rng = np.random.default_rng(seed)
        v = O.VocabularyArrays(10, 3, O.W_TF_IDF, O.S_L2, np.zeros(1, np.uint32), np.float32([2.5]), rng.integers(0, 256, (1, 32), dtype=np.uint8))
        return v, rng.integers(0, 256, (n, 32), dtype=np.uint8), 1
    return make


def _deeper_than_L(seed):
    def make():
        v = digit_tree(4, 6, seed)
        v = with_voc(v, L=3)
        rng = np.random.default_rng(seed)
        return v, digit_queries(4, rng.integers(0, 4, (700, 6))), 1
    return make


def _synth(k, L, n, seed, lu, prune=0.0, stop=0.0, weighting=O.W_TF_IDF, scoring=O.S_L1):
    def make():
        v = O.synth_vocabulary(k, L, seed=seed, weighting=weighting, scoring=scoring, prune=prune, stop=stop)
        return v, queries(v, n, seed + 1), lu
    return make


def _runs(n, lengths, fill=True, k=16, L=3, seed=0, weighting=O.W_TF_IDF, scoring=O.S_L1):
    """rows on consecutive leaves of a digit tree, the first runs of the given lengths, the rest of 1 to 9 rows (fill) or one run,
    in shuffled feature order"""
    def make():
        v = digit_tree(k, L, seed, weighting, scoring)
        rng = np.random.default_rng(seed)
        lens = list(lengths)
        while sum(lens) < n:
            lens.append(min(int(rng.integers(1, 10)) if fill else n, n - sum(lens)))
        assert len(lens) <= k ** L
        rows = np.concatenate([np.full(c, j) for j, c in enumerate(lens)]).astype(np.int64)
        rng.shuffle(rows)
        return v, digit_queries(k, leaf_paths(k, L, rows)), 0
    return make


def _one_differ(n, differ_at, stopped):
    """A digit tree of depth 3 whose first level-3 leaf has one child (one level deeper than L): with levelsup 0 a feature there
    files under the leaf, not under its word.  One feature goes there (index differ_at); `stopped`: its word has weight 0."""
    def make():
        k, L = 8, 3
        v = digit_tree(k, L, 5)
        p = first_leaf(k, L)
        child = np.append(v.child_num, np.uint32(0))
        child[p] = 1
        weight = np.append(v.weight, np.float32(0.0 if stopped else 3.25))
        desc = np.vstack([v.desc, v.desc[p][None]])
        v = with_voc(v, child_num=child, weight=weight, desc=desc)
        rng = np.random.default_rng(n)
        paths = rng.integers(0, k, (n, L))
        paths[(paths == 0).all(axis=1), 2] = 1
        paths[differ_at] = 0
        return v, digit_queries(k, paths), 0
    return make


def _odd_weights(seed):
    def make():
        v = O.synth_vocabulary(10, 3, seed=seed)
        f = queries(v, 3000, seed + 1)
        fw = O.bow_transform(v, f, 1)["f_word"]
        hit = np.unique(fw)
        w = v.weight.copy()
        w[hit[0]] = np.float32(-0.0)
        w[hit[1]] = np.float32(-1.5)
        w[hit[2]] = np.float32("nan")
        w[hit[3]] = np.float32(1e-40)               # subnormal
        w[hit[4]] = np.float32(2.0 ** -149)          # the smallest subnormal
        w[hit[5]] = np.float32(-3e-39)               # a negative subnormal
        return with_voc(v, weight=w), f, 1
    return make


def _stopped(all_but_one, weighting, scoring):
    def make():
        v = O.synth_vocabulary(10, 3, seed=13, weighting=weighting, scoring=scoring)
        f = queries(v, 1500, 14)
        w = np.zeros_like(v.weight)
        if all_but_one:
            fw = O.bow_transform(v, f, 1)["f_word"]
            w[fw[777]] = np.float32(0.625)
        return with_voc(v, weight=w), f, 1
    return make


ADVERSARIAL_W = np.float32(0.36225277)


def _adversarial():
    """IDF / L1 over 65 538 distinct words: the first word weighs 1, the second w, all the others 2^-54.  The reference's sequential
    norm absorbs every 2^-54; the tree keeps their sum (2^-38), and the second word's value comes out one float apart."""
    def make():
        k, L = 2, 17
        v = digit_tree(2, 17, 3, O.W_IDF, O.S_L1)
        n = 65538
        w = np.full(v.n_nodes, np.float32(2.0 ** -54), np.float32)
        p = first_leaf(k, L)
        w[p], w[p + 1] = np.float32(1.0), ADVERSARIAL_W
        return with_voc(v, weight=w), digit_queries(k, leaf_paths(k, L, np.arange(n))), 0
    return make


def _bound_inside(scoring):
    """2000 words, weights multiples of 2^-10, one word of weight 2^-20 (L1) or 2^-10 (L2: its square is 2^-20, the smallest lowest
    set bit of any term) and one large word that puts the total in [2^31, 2^32): every order of summation is exact, and the total
    is within a factor 2 of the bound."""
    def make():
        k, L = 2, 11
        v = digit_tree(k, L, 4, O.W_IDF, scoring)
        rng = np.random.default_rng(4)
        n = 2000
        p = first_leaf(k, L)
        w = v.weight.copy()
        w[p:p + n] = (rng.integers(205, 9216, n) / 1024.0).astype(np.float32)
        w[p + 7] = np.float32(2.0 ** -20 if scoring == O.S_L1 else 2.0 ** -10)
        w[p + 1500] = np.float32(2.0 ** 31 if scoring == O.S_L1 else 46341.0)
        return with_voc(v, weight=w), digit_queries(k, leaf_paths(k, L, np.arange(n))), 0
    return make


def _wide_idf(scoring):
    """idf weights log(N / n_i) of a large database span about 2^13: 2^-4 .. 2^9 here, 2000 rows.  Under L2 the squares keep 24
    significant bits over a span of 2^26 and the norm leaves the bound; under L1 it stays inside."""
    def make():
        v = O.synth_vocabulary(10, 4, seed=42, scoring=scoring)
        rng = np.random.default_rng(42)
        w = np.exp2(rng.uniform(-4.0, 9.0, v.n_nodes)).astype(np.float32)
        return with_voc(v, weight=w), queries(v, 2000, 43), 1
    return make


ROW_COUNTS =(1, 2, 3, 15, 17, 1023, 1024, 1025, 2047, 2049, 8191, 8192, 8193, 16385)

CASES = [
    # walk width and tree shape
    _c("k1_chain", _chain(12, 5, 300, 1), k=1, G=16, deeper_than_L=True),
    _c("k2", _walk_width(2, 9, 500, 2), k=2, G=16),
    _c("k15", _walk_width(15, 3, 900, 3, prune=True), k=15, G=16, fewer_children=True),
    _c("k16", _walk_width(16, 3, 900, 4), k=16, G=16),
    _c("k16_pruned", _walk_width(16, 3, 900, 5, prune=True), k=16, G=16, fewer_children=True),
    _c("k17", _walk_width(17, 3, 900, 6), k=17, G=32, hits_child_ge16=True),
    _c("k17_pruned", _walk_width(17, 3, 900, 7, prune=True), k=17, G=32, hits_child_ge16=True, fewer_children=True),
    _c("k31", _walk_width(31, 3, 900, 8, prune=True), k=31, G=32, hits_child_ge16=True, fewer_children=True),
    _c("k32", _walk_width(32, 3, 1000, 9), k=32, G=32, hits_child_ge16=True),
    _c("root_only", _root_only(100, 10), root_only=True, nw=1),
    _c("deeper_than_L", _deeper_than_L(11), deeper_than_L=True, same=False),
    _c("leaves_level1", _walk_width(20, 1, 300, 12), leaves_level1=True, G=32, hits_child_ge16=True),
    _c("nodes_1e6", _synth(10, 6, 3000, 13, 2), nodes_min=1_000_000, G=16),
    # levelsup on a balanced and on a pruned tree
    *[_c(f"lu_{name}_{kind}", _synth(10, 4, 1200, 20 + i, lu(4), prune=0.15 if kind == "pruned" else 0.0, stop=0.05), lu=name)
      for kind in ("balanced", "pruned")
      for i, (name, lu) in enumerate((("neg", lambda L: -2), ("0", lambda L: 0), ("1", lambda L: 1), ("L-1", lambda L: L - 1),
                                      ("L", lambda L: L), ("L+3", lambda L: L + 3)))],
    # row counts around the chunk and sort sizes (k 16 and 32: n*G not a multiple of 256 for most)
    *[_c(f"n{n}_k{k}", _synth(k, 3, n, n % 97 + k, 1, prune=0.1, stop=0.05), n=n, G=16 if k <= 16 else 32,
         **({"ng_mod256": True} if n * (16 if k <= 16 else 32) % 256 else {}))
      for n in ROW_COUNTS for k in ((10,) if n in (2, 15, 1024, 2047, 8192) else (10, 20))],
    # runs on chunk boundaries (per = 2 at n 1025, 16 at n 8193, 32 at n 16385)
    _c("runs_per2", _runs(1025, [2, 1, 3, 6, 5, 1, 1]), n=1025, per=2, run_starts_chunk=True, run_ends_chunk=True, run_spans=3),
    _c("runs_per16", _runs(8193, [16, 5, 27, 40, 3, 29, 7]), n=8193, per=16, in_smem=0, run_starts_chunk=True, run_ends_chunk=True,
       run_spans=3, same=True),
    _c("runs_per32_tf", _runs(16385, [32, 31, 97, 1, 200], weighting=O.W_TF, scoring=O.S_L2), n=16385, per=32, run_starts_chunk=True,
       run_ends_chunk=True, run_spans=7),
    _c("run_all_8193", _runs(8193, [], fill=False), n=8193, run_all=True, nw=1, in_smem=0),
    # the node sort
    _c("one_differ_last", _one_differ(5000, 4999 - 17, False), same=False, one_differ=True),
    _c("differ_stopped", _one_differ(5000, 3001, True), same=True, differ_stopped=True),
    # weights
    _c("odd_weights", _odd_weights(30), weights=("nan", "neg_zero", "negative", "subnormal")),
    *[_c(f"all_stopped_w{w}_s{s}", _stopped(False, w, s), nw=0) for w in range(4) for s in range(6)],
    *[_c(f"all_but_one_stopped_w{w}", _stopped(True, w, O.S_L2), nw=1) for w in range(4)],
    # the norm
    _c("norm_adversarial", _adversarial(), tree_differs=True, sequential=True, in_smem=0),
    _c("norm_inside_l1", _bound_inside(O.S_L1), bound_inside=True, sequential=False),
    _c("norm_inside_l2", _bound_inside(O.S_L2), bound_inside=True, sequential=False),
    _c("norm_l2_wide_idf", _wide_idf(O.S_L2), sequential=True),
    _c("norm_l1_wide_idf", _wide_idf(O.S_L1), sequential=False),
    _c("norm_l2_bench_like", _synth(10, 4, 2000, 40, 1, scoring=O.S_L2), sequential=False),
    _c("norm_l1_bench_like", _synth(10, 4, 2000, 41, 1), sequential=False),
]

BY_ID = {c.id: c for c in CASES}


def reference_defined(case):
    """The reference leaves the node id uninitialised for a negative levelsup and for a walk that ends above level L - levelsup."""
    v, f, lu = case.data
    if lu < 0:
        return False
    fw = O.bow_transform(v, f, lu)["f_word"]
    return bool(np.all(depths(v.k, fw) >= v.L - lu))


def check_reach(case, got_plan=None):
    """Assert that the case reaches its boundary, in the mirror's plan or in `got_plan` (the device's five values)."""
    v, f, lu = case.data
    n = len(f)
    ref = O.bow_transform(v, f, lu)
    want = device_plan(v, ref, n)
    p = got_plan if got_plan is not None else want
    g, sm, npad, npad_sorted, fl = p
    per = plan(v.k, n)[4]
    fold = norm_fold(v, ref)
    r = dict(case.reach)
    where = (case.id, p)
    vals = dict(G=g, in_smem=sm, npad=npad, npad_sorted=npad_sorted, per=per, same=bool(fl & 1), sequential=bool(fl & 2), k=v.k, n=n,
                nw=len(ref["words"]))
    for name, val in vals.items():
        if name in r:
            assert val == r[name], (name, val) + where
    fw, fn = ref["f_word"], ref["f_node"]
    d = depths(v.k, fw)
    if r.get("root_only"):
        assert v.n_nodes == 1, where
    if r.get("deeper_than_L"):
        assert d.max() > v.L, where
    if r.get("leaves_level1"):
        assert v.L == 1 and np.all(v.child_num[1:] == 0) and np.all(d == 1), where
    if "nodes_min" in r:
        assert v.n_nodes >= r["nodes_min"], where
    if r.get("hits_child_ge16") or r.get("fewer_children"):
        ge16 = fewer = False
        for x in np.unique(fw):
            while x > 0:
                par = (x - 1) // v.k
                ge16 |= (x - 1) % v.k >= 16
                fewer |= 0 < v.child_num[par] < v.k
                x = par
        if r.get("hits_child_ge16"):
            assert ge16, where
        if r.get("fewer_children"):
            assert fewer, where
    if "lu" in r:
        assert lu == {"neg": -2, "0": 0, "1": 1, "L-1": v.L - 1, "L": v.L, "L+3": v.L + 3}[r["lu"]], where
    if r.get("ng_mod256"):
        assert n * g % WALK_THREADS != 0, where
    heads, ends = fold["heads"], fold["ends"]
    if r.get("run_starts_chunk"):
        assert any(h > 0 and h % per == 0 and e - h > 1 for h, e in zip(heads, ends)), where
    if r.get("run_ends_chunk"):
        assert any(e % per == 0 and e - h > 1 and h // per != (e - 1) // per for h, e in zip(heads, ends)), where
    if "run_spans" in r:
        assert max((e - 1) // per - h // per + 1 for h, e in zip(heads, ends)) >= r["run_spans"], where
    if r.get("run_all"):
        assert len(heads) == 1 and ends[0] == n, where
    with np.errstate(invalid="ignore"):
        live = v.weight[fw] > 0
    differ = np.nonzero(fw != fn)[0]
    if r.get("one_differ"):
        dl = differ[live[differ]]
        assert len(dl) == 1 and dl[0] % RED_THREADS != 0, where
        kw, kf = live_keys(v, ref)
        pos = int(np.nonzero(kf == dl[0])[0][0])
        assert pos // per == (len(kw) - 1) // per, where
    if r.get("differ_stopped"):
        assert len(differ) >= 1 and not live[differ].any() and (fl & 1), where
    for kind in r.get("weights", ()):
        w = v.weight[fw]
        with np.errstate(invalid="ignore"):
            hit = {"neg_zero": (w == 0) & np.signbit(w), "negative": w < 0, "nan": np.isnan(w),
                   "subnormal": (w != 0) & (np.abs(w) < np.finfo(np.float32).tiny)}[kind]
        assert hit.any(), (kind,) + where
    if r.get("tree_differs"):
        assert not np.array_equal(normalise(v, fold, fold["tree"]), ref["values"]), where
    if r.get("bound_inside"):
        q = fold["q"]
        assert math.ldexp(1.0, q + 51) <= fold["tree"] < math.ldexp(1.0, q + 52) and fold["tree"] == fold["seq"], where
    return p
