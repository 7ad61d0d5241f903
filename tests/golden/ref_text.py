"""TEST INFRASTRUCTURE — run the UNMODIFIED reference ``dask_ml/feature_extraction/text.py`` without dask.

    BKM_REFERENCE=<dask-ml checkout> python tests/golden/ref_text.py   # regenerates tests/golden/ref_text_*.npz

``ref_shim.install()`` provides the eager stand-in for dask.array; the reference's HashingVectorizer also needs
``dask.is_dask_collection``, a ``dask.bag`` module (its ``Bag`` is only tested with isinstance) and a ``map_blocks``
that keeps the scipy.sparse blocks its transformer returns (``ref_encoders.Blocks``).  The reference's file is then
loaded with importlib, byte for byte.  Each case records the documents, their chunks, the parameters and the CSR of the
reference's blocks stacked; a 2-D array records the reference's error.  tests/test_text_host.py and
tests/test_gpu_text.py replay the fixtures; neither needs the reference checkout.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import scipy.sparse

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ref_shim  # noqa: E402
from ref_encoders import Blocks  # noqa: E402


def install():
    ref = ref_shim.install()
    Array = ref.da.Array
    dask = sys.modules["dask"]
    dask.is_dask_collection = lambda x: isinstance(x, Array)
    db = types.ModuleType("dask.bag")

    class Bag(object):
        pass

    db.Bag = Bag
    dask.bag = db
    sys.modules["dask.bag"] = db

    def map_blocks(self, func, *args, **kwargs):
        for k in ("dtype", "chunks", "new_axis", "drop_axis"):
            kwargs.pop(k, None)
        return Blocks([func(b, *args, **kwargs) for b in self.blocks])

    Array.map_blocks = map_blocks
    spec = importlib.util.spec_from_file_location(
        "dask_ml.feature_extraction.text", os.path.join(ref_shim.REF, "dask_ml", "feature_extraction", "text.py"))
    text = importlib.util.module_from_spec(spec)
    sys.modules["dask_ml.feature_extraction.text"] = text
    spec.loader.exec_module(text)
    return ref, text


def main():
    ref, text = install()
    from test_text_host import JUNK_FOOD_DOCS, word_docs

    cases = [
        ("ref_text_junk", list(JUNK_FOOD_DOCS), (3, 3), {}),
        ("ref_text_ngram_l1_f32", word_docs(200, 21), (70, 70, 60),
         dict(ngram_range=[1, 2], norm="l1", dtype="float32")),
        ("ref_text_binary_16", word_docs(120, 22) + ["", "a", "Zz zz ZZ"], (50, 73),
         dict(n_features=16, alternate_sign=False, binary=True, norm=None)),
    ]
    manifest = {"reference": "dask_ml/feature_extraction/text.py", "cases": []}
    for name, docs, chunks, params in cases:
        kw = dict(params)
        if "ngram_range" in kw:
            kw["ngram_range"] = tuple(kw["ngram_range"])
        if "dtype" in kw:
            kw["dtype"] = np.dtype(kw["dtype"]).type
        X = ref.da.from_array(np.array(docs, dtype=object), chunks=(chunks,))
        out = text.HashingVectorizer(**kw).transform(X)
        M = scipy.sparse.csr_matrix(out.compute())
        np.savez_compressed(os.path.join(HERE, name + ".npz"), docs=np.array(docs, dtype=str),
                            chunks=np.array(chunks, dtype=np.int64), indptr=M.indptr.astype(np.int64),
                            indices=M.indices.astype(np.int64), data=M.data)
        manifest["cases"].append({"file": name + ".npz", "params": params, "blocks": len(out.blocks),
                                  "block_type": type(out.blocks[0]).__name__})
    try:
        text.HashingVectorizer().transform(ref.da.from_array(np.array([["a b"], ["c d"]], dtype=object), chunks=(1,)))
        manifest["error_2d"] = None
    except ValueError as e:
        manifest["error_2d"] = str(e)
    with open(os.path.join(HERE, "REF_TEXT_MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
