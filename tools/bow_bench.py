"""Times the bag-of-words transform (gb_bow_transform, host buffers in and out) against the reference's Vocabulary::transform
(oracle/_ref when present, else the oracle port) on 2000 descriptors -- the "Trans ORB-4" line of doc/doxygen/4_2_tools.dox:43."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import oracle
from oracle import oracle as O
from gslam_b200.api import Context, Vocabulary

ctx = Context(0)
for k, L in ((10, 4), (10, 5), (10, 6)):
    v = O.synth_vocabulary(k, L, seed=1)
    dv = Vocabulary(ctx, v.k, v.L, v.weighting, v.scoring, v.child_num, v.weight, v.desc)
    rng = np.random.default_rng(0)
    f = v.desc[rng.integers(1, v.n_nodes, 2000)] ^ np.packbits(rng.random((2000, 256)) < 0.05, axis=1)
    got = dv.transform(f, 2)
    want = O.bow_transform(v, f, 2)
    ok = all(np.array_equal(got[x], want[x]) for x in ("words", "values", "fv_node", "fv_feat"))
    for _ in range(5):
        dv.transform(f, 2)
    t0 = time.perf_counter()
    for _ in range(200):
        dv.transform(f, 2)
    t_gpu = (time.perf_counter() - t0) / 200
    if oracle.have_ref():
        R = O.RefVocabulary.from_arrays(v)
        t_ref = R.transform(f, 2, repeat=20)["seconds"]; kind = "reference (oracle/_ref)"
        R.close()
    else:
        t0 = time.perf_counter(); O.bow_transform(v, f, 2); t_ref = time.perf_counter() - t0; kind = "oracle port"
    print(f"k={k} L={L} ({v.n_nodes} nodes): parity {ok}; GPU {t_gpu * 1e6:.1f} us per 2000-descriptor transform (host in, host out, python call included); "
          f"{kind} {t_ref * 1e6:.1f} us", flush=True)
    dv.close()
