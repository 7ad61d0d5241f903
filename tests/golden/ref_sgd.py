"""TEST INFRASTRUCTURE — run the UNMODIFIED reference SGD family (``dask_ml/linear_model/{stochastic_gradient,
perceptron,passive_aggressive}.py`` on ``dask_ml/_partial.py``) without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_sgd.py   # regenerates tests/golden/ref_sgd_*.npz

``ref_minibatch.install()`` provides the eager dask stand-in and the reference's ``_utils.py`` / ``_partial.py``.  The
reference imports ``sklearn.linear_model.stochastic_gradient``, which scikit-learn has since renamed
``_stochastic_gradient``: the old name is aliased to the new module.  The three reference files are then loaded with
importlib, byte for byte.  Their ``fit`` calls the installed scikit-learn's ``partial_fit`` once per block (with
``classes`` for the classifiers), in the order the global numpy RNG shuffles the blocks into; each case seeds that RNG
and records the order.  The cases are the reference tests' estimators and parameters
(tests/linear_model/test_{stochastic_gradient,perceptron,passive_aggressive}.py), the PassiveAggressive regressor,
and multi-block, multi-class and averaged cases.  tests/test_sgd_host.py and tests/test_gpu_sgd.py replay the
fixtures; neither needs the reference checkout.
"""
import json
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_minibatch  # noqa: E402
import ref_shim  # noqa: E402


def install():
    ref, _mb = ref_minibatch.install()
    import sklearn.linear_model
    import sklearn.linear_model._stochastic_gradient as sg

    sys.modules["sklearn.linear_model.stochastic_gradient"] = sg
    sklearn.linear_model.stochastic_gradient = sg
    # 1-D arrays (y) are keyed (name, i) in the block-wise graph, 2-D ones (name, i, 0)
    ref.da.Array.dask = property(lambda self: {((self.name, i, 0) if self.ndim == 2 else (self.name, i)): b
                                               for i, b in enumerate(self.blocks)})
    root = os.path.join(ref_shim.REF, "dask_ml", "linear_model")
    pkg = types.ModuleType("dask_ml.linear_model")
    pkg.__path__ = [root]
    sys.modules["dask_ml.linear_model"] = pkg
    mods = {}
    for name in ("stochastic_gradient", "perceptron", "passive_aggressive"):
        mods[name] = _load("dask_ml.linear_model." + name, os.path.join(root, name + ".py"))
    return ref, mods


def _load(name, path):
    import importlib.util

    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def _classification(n, d, k, seed):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    W = rng.standard_normal((d, k))
    return X, np.argmax(X @ W + 0.5 * rng.standard_normal((n, k)), axis=1)


def _regression(n, d, seed):
    rng = np.random.RandomState(seed)
    X = rng.standard_normal((n, d))
    return X, X @ rng.standard_normal(d) + 0.1 * rng.standard_normal(n)


def cases():
    """name -> (module, class, X, y, block rows, constructor keywords)."""
    Xc, yc = _classification(100, 20, 2, 1)             # the reference tests' single-chunk problems
    Xr, yr = _regression(100, 20, 2)
    X3, y3 = _classification(1200, 10, 3, 3)
    X20, y20 = _classification(1000, 12, 20, 4)
    Xm, ym = _regression(900, 8, 5)
    return {
        "ref_sgd_classifier_basic": ("stochastic_gradient", "PartialSGDClassifier", Xc, yc, 100,
                                     dict(classes=[0, 1], random_state=0, max_iter=1000, tol=1e-3)),
        "ref_sgd_regressor_basic": ("stochastic_gradient", "PartialSGDRegressor", Xr, yr, 100,
                                    dict(random_state=0, max_iter=1000, tol=1e-3)),
        "ref_sgd_perceptron_basic": ("perceptron", "PartialPerceptron", Xc, yc, 100,
                                     dict(classes=[0, 1], max_iter=1000, tol=1e-3)),
        "ref_sgd_pa_classifier_basic": ("passive_aggressive", "PartialPassiveAggressiveClassifier", Xc, yc, 100,
                                        dict(classes=[0, 1], random_state=0, max_iter=100, tol=1e-3)),
        "ref_sgd_pa_regressor_blocks": ("passive_aggressive", "PartialPassiveAggressiveRegressor", Xm, ym, 200,
                                        dict(random_state=0)),
        "ref_sgd_classifier_3_blocks": ("stochastic_gradient", "PartialSGDClassifier", X3, y3, 250,
                                        dict(classes=[0, 1, 2], random_state=7, penalty="elasticnet")),
        "ref_sgd_classifier_20_average": ("stochastic_gradient", "PartialSGDClassifier", X20, y20, 300,
                                          dict(classes=list(range(20)), random_state=8, average=True,
                                               loss="modified_huber")),
        "ref_sgd_regressor_blocks_average": ("stochastic_gradient", "PartialSGDRegressor", Xm, ym, 200,
                                             dict(random_state=9, average=100, loss="huber")),
    }


def main():
    ref, mods = install()
    manifest = {}
    for ci, (name, (mod, cls, X, y, rows, kw)) in enumerate(cases().items()):
        seed = 200 + ci
        nb = (len(X) + rows - 1) // rows
        np.random.seed(seed)
        order = list(range(nb))
        np.random.shuffle(order)                         # the shuffle the reference's fit draws, replayed
        np.random.seed(seed)
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            est = getattr(mods[mod], cls)(**kw)
        deprecation = [str(w.message) for w in rec if issubclass(w.category, FutureWarning)]
        Xd = ref.da.from_array(X, chunks=(rows, X.shape[1]))
        yd = ref.da.from_array(y, chunks=(rows,))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            est.fit(Xd, yd)
        params = {k: v for k, v in kw.items()}
        np.savez_compressed(os.path.join(HERE, name + ".npz"), X=X, y=y, rows=rows, seed=seed, order=np.array(order),
                            coef=np.asarray(est.coef_), intercept=np.atleast_1d(est.intercept_),
                            t=np.float64(est.t_))
        manifest[name] = dict(module=mod, cls=cls, n=int(X.shape[0]), d=int(X.shape[1]), block_rows=rows, seed=seed,
                              params=params, order=order, t=float(est.t_), deprecation=deprecation)
        print(name, manifest[name], flush=True)
    import sklearn

    with open(os.path.join(HERE, "REF_SGD_MANIFEST.json"), "w") as f:
        json.dump({"reference": "mrocklin/dask-ml @ 0310a90 _partial.py + linear_model/{stochastic_gradient,"
                                "perceptron,passive_aggressive}.py run through tests/golden/ref_sgd.py with "
                                "scikit-learn %s" % sklearn.__version__, "cases": manifest}, f, indent=1)


if __name__ == "__main__":
    main()
