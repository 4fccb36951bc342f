"""Throughput of the percolator (tb.Percolator / trn_percolate): a registry of bench.py's and2 and tree8 query shapes plus 2-3-term
phrases over the 4096-term vocabulary, with term_cost = the synthetic index's document frequencies (bench.synth_dfs), against documents of
tokens drawn from the same Zipf(1) rank distribution.  Reports the registration time, the anchor entries, candidates and matches per
document, the device time of the count and the write pass (CUDA events around the kernels), documents/s over the whole call and candidate
evaluations/s over the count pass; then runs the reference's own percolator_query::match (oracle/_ref/libtrinity_ref_perc.so, one host
thread, each document against every query) over a prefix of the documents, compares every result of that prefix and prints its rate
beside the device's.  The card name and its power limit are printed with the numbers (read-only nvidia-smi query).

With query-log-like terms most documents hold the common terms, so the result grows as documents x queries x match rate: the defaults
keep one call's result well under 1 GB.

    python scripts/microbench_percolate.py [--nq 100000] [--ndocs 4000] [--doc-len 64] [--ref-docs 8] [--steps 3]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import bench  # noqa: E402
import trinity_b200 as tb  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def phrases(nq, nterms, seed=0xFACE):
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, nterms + 1)
    w /= w.sum()
    return ['"' + " ".join(f"t{r + 1:04d}" for r in rng.choice(nterms, size=int(rng.integers(2, 4)), p=w)) + '"' for _ in range(nq)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=100_000, help="queries of each shape (and2, tree8, phrase)")
    ap.add_argument("--ndocs", type=int, default=4000)
    ap.add_argument("--doc-len", type=int, default=64)
    ap.add_argument("--ref-docs", type=int, default=8, help="documents of the prefix run through the reference and compared")
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    out = {"card": card()}
    print(json.dumps(out), flush=True)
    names = [f"t{r:04d}" for r in range(1, args.nterms + 1)]
    tdict = tb.TermDictionary(names)
    texts = bench.gen_queries("and2", args.nq, args.nterms)[0] + bench.gen_queries("tree8", args.nq, args.nterms)[0] + phrases(args.nq, args.nterms)
    trees = [tb.parse_query(q, tdict) for q in texts]
    cost = np.minimum(bench.synth_dfs(100_000_000, args.nterms), 0xFFFFFFFF).astype(np.uint32)
    rng = np.random.default_rng(0xD0C5)
    w = 1.0 / np.arange(1, args.nterms + 1)
    w /= w.sum()
    docs = [rng.choice(args.nterms, size=args.doc_len, p=w).astype(np.uint32) for _ in range(args.ndocs)]

    t0 = time.perf_counter()
    p = tb.Percolator(trees, nterms=args.nterms, term_cost=cost)
    reg_s = time.perf_counter() - t0
    info = p.info()
    p.percolate(docs)  # warm-up
    best = None
    for _ in range(args.steps):
        r = p.percolate(docs)
        if best is None or r.total_ms < best.total_ms:
            best = r
    res = {"queries": len(trees), "documents": args.ndocs, "doc_tokens": args.doc_len, "register_s": round(reg_s, 3), "anchor_entries": info["anchor_entries"],
           "never": info["never"], "registry_mb": round(info["device_bytes"] / 1e6, 1), "candidates_per_doc": round(best.candidates / args.ndocs, 1),
           "matches_per_doc": round(best.total / args.ndocs, 1), "result_mb": round(best.total * 4 / 1e6, 1), "dense_docs": best.dense_docs,
           "count_ms": round(best.count_ms, 3), "write_ms": round(best.write_ms, 3), "call_ms": round(best.total_ms, 3),
           "docs_per_s_call": round(args.ndocs / (best.total_ms / 1e3)), "candidate_evals_per_s_count_pass": round(best.candidates / (best.count_ms / 1e3))}
    print(json.dumps({"device": res}), flush=True)

    from percutil import RefPercolator
    nref = min(args.ref_docs, args.ndocs)
    ref = RefPercolator([(q, 0, 0) for q in texts], vocab=names)
    t0 = time.perf_counter()
    want = ref.run(docs[:nref])
    ref_s = time.perf_counter() - t0
    parity = all(np.array_equal(best.document(d), want[d]) for d in range(nref))
    out.update(device=res, reference={"documents": nref, "s_per_doc_1_thread": round(ref_s / max(1, nref), 3),
                                      "docs_per_s_1_thread": round(nref / ref_s, 2) if ref_s else None,
                                      "pair_evals_per_s_1_thread": round(nref * len(texts) / ref_s) if ref_s else None, "parity": bool(parity)})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
