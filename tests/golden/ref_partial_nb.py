"""TEST INFRASTRUCTURE — run the UNMODIFIED reference PartialMultinomialNB / PartialBernoulliNB
(``dask_ml/naive_bayes.py`` on ``dask_ml/_partial.py``) without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_partial_nb.py   # regenerates tests/golden/ref_partial_nb_*.npz

``ref_minibatch.install()`` provides the eager dask stand-in and the reference's ``_utils.py`` / ``_partial.py``; the
reference's ``naive_bayes.py`` is then loaded with importlib, byte for byte (its GaussianNB is not used here, so the
extra stand-ins of ``ref_naive_bayes.py`` are not needed).  The reference's ``fit`` calls the installed scikit-learn's
``partial_fit`` once per block with ``classes``, in the order the global numpy RNG shuffles the blocks into; each case
seeds that RNG and records the order, the learned attributes, the predictions of the reference's ``predict`` and the
log-probabilities on X.  Cases marked sparse are replayed from a scipy CSR copy of X (the counts of integer data do
not depend on the form of X).  tests/test_partial_nb_host.py replays the fixtures without the reference checkout.
"""
import importlib.util
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_minibatch  # noqa: E402
import ref_shim  # noqa: E402


def install():
    ref, _mb = ref_minibatch.install()
    # 1-D arrays (y) are keyed (name, i) in the block-wise graph, 2-D ones (name, i, 0)
    ref.da.Array.dask = property(lambda self: {((self.name, i, 0) if self.ndim == 2 else (self.name, i)): b
                                               for i, b in enumerate(self.blocks)})
    path = os.path.join(ref_shim.REF, "dask_ml", "naive_bayes.py")
    spec = importlib.util.spec_from_file_location("dask_ml.naive_bayes", path)
    m = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.naive_bayes"] = m
    spec.loader.exec_module(m)
    return ref, m


def _counts(n, d, K, seed):
    rng = np.random.RandomState(seed)
    X = rng.poisson(1.5, size=(n, d)).astype(np.float64) * (rng.uniform(size=(n, d)) < 0.4)
    return X, rng.randint(0, K, size=n)


def cases():
    """name -> (class, X, y, block rows, constructor keywords, replay as CSR)."""
    Xa, ya = _counts(600, 20, 3, 1)
    Xb, yb = _counts(1000, 30, 5, 2)
    rng = np.random.RandomState(3)
    Xc = rng.standard_normal((800, 10))
    yc = (Xc[:, 0] + 0.5 * rng.standard_normal(800) > 0).astype(np.int64)
    Xd, yd = _counts(900, 16, 3, 4)
    return {
        "ref_partial_nb_mnb_basic": ("PartialMultinomialNB", Xa, ya, 150, dict(classes=[0, 1, 2]), False),
        "ref_partial_nb_mnb_alpha_csr": ("PartialMultinomialNB", Xb, yb, 250,
                                         dict(classes=[0, 1, 2, 3, 4], alpha=0.5, fit_prior=False), True),
        "ref_partial_nb_bnb_basic": ("PartialBernoulliNB", Xc, yc, 200, dict(classes=[0, 1]), False),
        "ref_partial_nb_bnb_threshold_csr": ("PartialBernoulliNB", Xd, yd + 1, 300,
                                             dict(classes=[1, 2, 3], binarize=1.5), True),
    }


def main():
    ref, nb = install()
    manifest = {}
    for ci, (name, (cls, X, y, rows, kw, sparse)) in enumerate(cases().items()):
        seed = 300 + ci
        nblk = (len(X) + rows - 1) // rows
        np.random.seed(seed)
        order = list(range(nblk))
        np.random.shuffle(order)                         # the shuffle the reference's fit draws, replayed
        np.random.seed(seed)
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            est = getattr(nb, cls)(**kw)
        deprecation = [str(w.message) for w in rec if issubclass(w.category, FutureWarning)]
        Xd = ref.da.from_array(X, chunks=(rows, X.shape[1]))
        yd = ref.da.from_array(y, chunks=(rows,))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            est.fit(Xd, yd)
            pred = np.asarray(est.predict(X))
            lp = est.predict_log_proba(X)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), X=X, y=y, rows=rows, seed=seed, order=np.array(order),
                            feature_count=est.feature_count_, class_count=est.class_count_,
                            feature_log_prob=est.feature_log_prob_, class_log_prior=est.class_log_prior_,
                            predict=pred, predict_log_proba=lp)
        manifest[name] = dict(cls=cls, n=int(X.shape[0]), d=int(X.shape[1]), block_rows=rows, seed=seed, params=kw,
                              sparse=sparse, order=order, class_count=[float(c) for c in est.class_count_],
                              deprecation=deprecation)
        print(name, manifest[name], flush=True)
    import sklearn

    with open(os.path.join(HERE, "REF_PARTIAL_NB_MANIFEST.json"), "w") as f:
        json.dump({"reference": "mrocklin/dask-ml @ 0310a90 _partial.py + naive_bayes.py run through "
                                "tests/golden/ref_partial_nb.py with scikit-learn %s" % sklearn.__version__,
                   "cases": manifest}, f, indent=1)


if __name__ == "__main__":
    main()
