"""HashingVectorizer on the H100: a seeded Zipf-vocabulary ASCII corpus of about 1 GB in blocks of 2M documents, at
ngram_range (1, 1) and (1, 2).

    python tests/text_bench.py [--gb 1.0] [--docs-per-block 2000000] [--repeats 3] [--out results/text_bench.json]

Reported per ngram_range, from CUDA events and host clocks around work that ends in a synchronise:
  * device: the three passes alone (bkm_text_tokens_chunk, _hash_chunk, _write_chunk with their two count reads) on one
    block already packed on the device, against the HBM floor of one read of its bytes and one write of its CSR
    (indptr, int64 indices, data) at 3.35 TB/s;
  * pack_h2d: host routing and packing of one block plus its host-to-device copy;
  * transform: HashingVectorizer.transform of the whole corpus, every block, ending in a synchronise;
  * scikit-learn's transform of a subset of documents, its rate, and a bit-for-bit comparison of its CSR with the
    device result of the same documents.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse
import sklearn.feature_extraction.text
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dask_ml_b200 import ChunkedArray  # noqa: E402
from dask_ml_b200.cluster import k_means as _km  # noqa: E402
from dask_ml_b200.feature_extraction import HashingVectorizer, text  # noqa: E402

HBM = 3.35e12


def corpus(total_bytes, seed=0, vocab=50000, mean_words=80):
    """Documents of Zipf(1.1)-ranked words of 2-12 lowercase or capitalised letters, each followed by ' ' or, one time
    in eight, ', ' or '. '."""
    rng = np.random.RandomState(seed)
    letters = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    words = [bytes(letters[rng.randint(0, 26, L)]).decode() for L in rng.randint(2, 13, vocab)]
    words = [w.capitalize() if i % 7 == 0 else w for i, w in enumerate(words)]
    entries = np.array([w + s for s in (" ", " ", " ", " ", " ", " ", ", ", ". ") for w in words], dtype=object)
    elen = np.fromiter(map(len, entries), dtype=np.int64, count=entries.size)

    def draw(m):
        return np.minimum(rng.zipf(1.1, m) - 1, vocab - 1) + vocab * rng.randint(0, 8, m)

    n_words = int(total_bytes / elen[draw(1 << 20)].mean())
    ids = draw(n_words)
    big = "".join(entries[ids].tolist())
    sizes = np.maximum(1, rng.poisson(mean_words, n_words // mean_words + 1))
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    cuts = np.concatenate([[0], np.cumsum(elen[ids])])[bounds[bounds <= n_words]]
    return [big[a:b] for a, b in zip(cuts[:-1].tolist(), cuts[1:].tolist())]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def timed(fn, repeats):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(repeats)]
    out = None
    for a, b in ev:
        a.record()
        out = fn()
        b.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) / 1e3 for a, b in ev], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=1.0)
    ap.add_argument("--docs-per-block", type=int, default=2_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sk-docs", type=int, default=20000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "text_bench needs a GPU"
    t0 = time.perf_counter()
    docs = corpus(int(args.gb * 1e9))
    gen_s = time.perf_counter() - t0
    nbytes = sum(map(len, docs))
    X = ChunkedArray.from_array(np.array(docs, dtype=object), args.docs_per_block)
    res = {"card": card(), "docs": len(docs), "bytes": nbytes, "blocks": len(X.blocks), "corpus_s": gen_s, "runs": []}
    be = _km._get_backend()
    first = X.blocks[0].tolist()
    for ngram in ((1, 1), (1, 2)):
        est = HashingVectorizer(ngram_range=ngram)
        cfg = text.device_config(est)
        r = {"ngram_range": list(ngram)}

        def pack_h2d():
            dev, _, _, joined = text.route(first)
            buf, off = text.pack(dev, joined)
            return torch.from_numpy(buf).to(be.device), torch.from_numpy(off).to(be.device)

        pack_h2d()
        t = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            s = time.perf_counter()
            buf_d, off_d = pack_h2d()
            torch.cuda.synchronize()
            t.append(time.perf_counter() - s)
        r["pack_h2d_s"] = t
        text.device_rows(be, buf_d, off_d, cfg)                       # warm-up
        dt, (ip, col, val) = timed(lambda: text.device_rows(be, buf_d, off_d, cfg), args.repeats)
        nnz = int(ip[-1].item())
        floor_bytes = buf_d.numel() + off_d.numel() * 8 + nnz * (8 + val.element_size())
        r.update(device_s=dt, block_docs=len(first), block_bytes=int(buf_d.numel()), block_nnz=nnz,
                 hbm_floor_s=floor_bytes / HBM, device_over_floor=min(dt) / (floor_bytes / HBM),
                 device_gb_per_s=buf_d.numel() / min(dt) / 1e9)
        est.transform(ChunkedArray(X.blocks[:1]))                     # warm-up of the whole path
        t = []
        for _ in range(args.repeats):
            torch.cuda.synchronize()
            s = time.perf_counter()
            out = est.transform(X)
            torch.cuda.synchronize()
            t.append(time.perf_counter() - s)
        r["transform_s"] = t
        r["transform_mb_per_s"] = nbytes / min(t) / 1e6
        sub = first[: args.sk_docs]
        s = time.perf_counter()
        want = sklearn.feature_extraction.text.HashingVectorizer(ngram_range=ngram).transform(sub)
        sk_s = time.perf_counter() - s
        got = scipy.sparse.csr_matrix(est.transform(ChunkedArray([np.array(sub, dtype=object)])).compute())
        same = (np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
                and np.array_equal(got.data.view(np.uint8), want.data.view(np.uint8)))
        # the whole-corpus device result, first block's first rows, against the same scikit-learn rows
        b0, m = out.blocks[0], len(sub)
        crow = b0.crow_indices()[: m + 1].cpu().numpy()
        head = scipy.sparse.csr_matrix((b0.values()[: crow[-1]].cpu().numpy(), b0.col_indices()[: crow[-1]].cpu().numpy(),
                                        crow), shape=(m, b0.shape[1]))
        same_full = (np.array_equal(head.indptr, want.indptr) and np.array_equal(head.indices, want.indices)
                     and np.array_equal(head.data.view(np.uint8), want.data.view(np.uint8)))
        r.update(sklearn_docs=len(sub), sklearn_s=sk_s, sklearn_mb_per_s=sum(map(len, sub)) / sk_s / 1e6,
                 bit_identical=bool(same and same_full))
        res["runs"].append(r)
        print(json.dumps(r), flush=True)
        del out, ip, col, val, buf_d, off_d
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}))
    assert all(r["bit_identical"] for r in res["runs"])


if __name__ == "__main__":
    main()
