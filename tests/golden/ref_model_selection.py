"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/model_selection/_split.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_model_selection.py   # regenerates ref_split_*.npz

``ref_shim.install()`` provides the eager stand-in for dask (``dask.delayed``, ``da.from_delayed`` and ``da.concatenate``
included).  Two more pieces are added here:
  * ``sklearn.model_selection._split._validate_shuffle_split_init``, removed from scikit-learn in 0.24: its constructor
    checks restated (both sizes None, a float size >= 1, a size that is neither float nor int, a float sum above 1);
  * a recorder around the module's ``_generate_idx``, which sees what the reference hands every block: the block's rows,
    its seed and its ``(n_train, n_test)``.
The reference file is then loaded with importlib, byte for byte.  Each case records those per-block values and the row
chunks of the index arrays and of the split outputs; the manifest also records the text of the reference's errors.
The permutation itself is not recorded: the package replaces numpy's serial shuffle by its own keyed bijection
(DESIGN.md A26).  tests/test_model_selection_host.py replays the fixtures without the reference checkout.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402


def _validate_shuffle_split_init(test_size, train_size):
    if test_size is None and train_size is None:
        raise ValueError("test_size and train_size can not both be None")
    for name, size in (("test_size", test_size), ("train_size", train_size)):
        if size is None:
            continue
        kind = np.asarray(size).dtype.kind
        if kind == "f":
            if size >= 1.0:
                raise ValueError("{}={} should be smaller than 1.0 or be an integer".format(name, size))
        elif kind != "i":
            raise ValueError("Invalid value for {}: {!r}".format(name, size))
    if (train_size is not None and test_size is not None and np.asarray(train_size).dtype.kind == "f"
            and np.asarray(test_size).dtype.kind == "f" and train_size + test_size > 1.0):
        raise ValueError("The sum of test_size and train_size = {}, should be smaller than 1.0. Reduce test_size "
                         "and/or train_size.".format(train_size + test_size))


def install():
    ref = ref_shim.install()
    import sklearn.model_selection._split as sk_split

    sk_split._validate_shuffle_split_init = _validate_shuffle_split_init
    root = os.path.join(ref_shim.REF, "dask_ml")
    pkg = types.ModuleType("dask_ml.model_selection")
    pkg.__path__ = [os.path.join(root, "model_selection")]
    sys.modules["dask_ml.model_selection"] = pkg
    path = os.path.join(root, "model_selection", "_split.py")
    spec = importlib.util.spec_from_file_location("dask_ml.model_selection._split", path)
    m = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.model_selection._split"] = m
    spec.loader.exec_module(m)
    calls = []
    original = m._generate_idx

    def recorder(n, seed, n_train, n_test):
        calls.append((int(n), int(seed), int(n_train), int(n_test)))
        return original(n, seed, n_train, n_test)

    m._generate_idx = recorder
    return ref, m, calls


def _rs(spec):
    return np.random.RandomState(spec["RandomState"]) if isinstance(spec, dict) else spec


CASES = {
    "ref_split_equal": dict(chunks=[50, 50, 50, 50], d=4, random_state=0, test_size=0.2),
    "ref_split_ragged": dict(chunks=[50, 50, 25], d=4, random_state=0),
    "ref_split_one_block": dict(chunks=[113], d=3, random_state=7, test_size=0.25),
    "ref_split_short_block": dict(chunks=[40, 40, 39, 2], d=2, random_state=3, test_size=0.5),
    "ref_split_train_only": dict(chunks=[64, 36], d=5, random_state=11, train_size=0.7),
    "ref_split_both": dict(chunks=[100, 60, 7], d=2, random_state=5, test_size=0.3, train_size=0.7),
    "ref_split_rs_instance": dict(chunks=[30, 30, 30], d=3, random_state={"RandomState": 42}, test_size=0.1),
    "ref_split_many_blocks": dict(chunks=[10] * 12 + [9], d=1, random_state=2 ** 31 - 1, test_size=0.4),
}

SHUFFLE_CASE = dict(chunks=[20, 20, 11], n_splits=3, test_size=0.25, random_state=9)

ERRORS = {
    "int_test_size": dict(fn="train_test_split", kw=dict(test_size=3)),
    "int_train_size": dict(fn="train_test_split", kw=dict(train_size=3)),
    "test_size_above_1": dict(fn="split", kw=dict(test_size=0.5, train_size=1.5)),
    "test_size_negative": dict(fn="train_test_split", kw=dict(test_size=-0.1)),
    "train_size_negative": dict(fn="train_test_split", kw=dict(train_size=-0.25)),
    "sum_not_1": dict(fn="train_test_split", kw=dict(test_size=0.3, train_size=0.3)),
    "both_none": dict(fn="ShuffleSplit", kw=dict(test_size=None, train_size=None)),
    "blockwise_not_bool": dict(fn="ShuffleSplit", kw=dict(blockwise="yes")),
    "blockwise_false": dict(fn="train_test_split", kw=dict(blockwise=False)),
    "shuffle_false": dict(fn="train_test_split", kw=dict(shuffle=False)),
    "unexpected_option": dict(fn="train_test_split", kw=dict(stratify=None)),
    "one_row_block": dict(fn="train_test_split", kw=dict(test_size=0.5), chunks=[10, 1]),
}


def run_error(m, da, spec):
    chunks = spec.get("chunks", [10, 10])
    X = da.from_array(np.arange(sum(chunks) * 2.0).reshape(-1, 2), chunks=(tuple(chunks), 2))
    if spec["fn"] == "ShuffleSplit":
        m.ShuffleSplit(**spec["kw"])
    elif spec["fn"] == "split":
        ss = m.ShuffleSplit(n_splits=1)
        for k, v in spec["kw"].items():               # past the constructor: the checks of the split itself
            setattr(ss, k, v)
        next(ss.split(X))
    else:
        m.train_test_split(X, **spec["kw"])


def main():
    ref, m, calls = install()
    da = ref.da
    manifest = {"reference": "mrocklin/dask-ml @ 0310a90 model_selection/_split.py run through "
                             "tests/golden/ref_model_selection.py", "cases": {}, "errors": {}}
    for name, case in CASES.items():
        chunks, d = case["chunks"], case["d"]
        n = sum(chunks)
        X = np.arange(n * d, dtype=np.float64).reshape(n, d)
        y = np.arange(n, dtype=np.int64)
        kw = {k: case[k] for k in ("test_size", "train_size") if k in case}
        del calls[:]
        out = m.train_test_split(da.from_array(X, chunks=(tuple(chunks), d)), da.from_array(y, chunks=(tuple(chunks),)),
                                 random_state=_rs(case["random_state"]), **kw)
        rec = np.array(calls, dtype=np.int64)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), chunks=np.array(chunks), seeds=rec[:, 1].astype(np.uint64),
                            block_rows=rec[:, 0], n_train=rec[:, 2], n_test=rec[:, 3],
                            train_chunks=np.array(out[0].chunks[0]), test_chunks=np.array(out[1].chunks[0]),
                            y_train_chunks=np.array(out[2].chunks[0]), y_test_chunks=np.array(out[3].chunks[0]))
        manifest["cases"][name] = dict(case, n_outputs=len(out), x_train_shape=list(out[0].shape),
                                       y_test_shape=list(out[3].shape))
        print(name, manifest["cases"][name], flush=True)
    # ShuffleSplit.split draws the seeds again from random_state at every split
    sc = SHUFFLE_CASE
    X = da.from_array(np.zeros((sum(sc["chunks"]), 2)), chunks=(tuple(sc["chunks"]), 2))
    del calls[:]
    ss = m.ShuffleSplit(n_splits=sc["n_splits"], test_size=sc["test_size"], random_state=sc["random_state"])
    idx_chunks = [[list(tr.chunks[0]), list(te.chunks[0])] for tr, te in ss.split(X)]
    rec = np.array(calls, dtype=np.int64).reshape(sc["n_splits"], len(sc["chunks"]), 4)
    np.savez_compressed(os.path.join(HERE, "ref_split_shufflesplit.npz"), seeds=rec[:, :, 1].astype(np.uint64),
                        n_train=rec[:, :, 2], n_test=rec[:, :, 3], idx_chunks=np.array(idx_chunks))
    manifest["shufflesplit"] = dict(sc, n_splits_reported=ss.get_n_splits())
    for name, spec in ERRORS.items():
        try:
            run_error(m, da, spec)
            manifest["errors"][name] = None
        except Exception as e:
            manifest["errors"][name] = dict(spec, type=type(e).__name__, message=str(e))
        print(name, manifest["errors"][name], flush=True)
    with open(os.path.join(HERE, "REF_MODEL_SELECTION_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
