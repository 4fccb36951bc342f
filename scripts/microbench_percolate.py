"""Throughput of the percolator (tb.Percolator / trn_percolate): a registry of bench.py's and2 and tree8 query shapes plus 2-3-term
phrases over the 4096-term vocabulary, with term_cost = the synthetic index's document frequencies (bench.synth_dfs), against documents of
tokens drawn from the same Zipf(1) rank distribution.  Reports the registration time, the anchor entries, candidates and matches per
document, the device time of the count and the write pass (CUDA events around the kernels), documents/s over the whole call and candidate
evaluations/s over the count pass; then runs the reference's own percolator_query::match (oracle/_ref/libtrinity_ref_perc.so, one host
thread, each document against every query) over a prefix of the documents, compares every result of that prefix and prints its rate
beside the device's.  The card name and its power limit are printed with the numbers (read-only nvidia-smi query).

With query-log-like terms most documents hold the common terms, so the result grows as documents x queries x match rate: the defaults
keep one call's result well under 1 GB.

--churn measures the in-place updates (Percolator.add / remove) instead: after the registration it adds 1, 1 000 and 30 000 queries of
the same shapes and removes 1 000 and 30 000 random live ones, each timed on the host clock around the call (which ends in a
synchronise) and with the CUDA events around its device work (uploads, program copies, rebuild kernels); then it times trn_percolate on the
churned registry and on a fresh registration of the same live set, alternating them, and compares the churned registry's results with
the reference's over the live query texts on the prefix.

    python scripts/microbench_percolate.py [--nq 100000] [--ndocs 4000] [--doc-len 64] [--ref-docs 8] [--steps 3] [--churn]
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
    ap.add_argument("--churn", action="store_true", help="time adds and removes, and percolate on the churned registry against a fresh one")
    args = ap.parse_args()
    if args.churn:
        return churn(args)
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


def workload(nq, nterms, seed):
    """nq queries of each shape (and2, tree8, phrase), drawn from the seed"""
    return (bench.gen_queries("and2", nq, nterms, seed=seed)[0] + bench.gen_queries("tree8", nq, nterms, seed=seed + 1)[0]
            + phrases(nq, nterms, seed=seed + 2))


def churn(args):
    out = {"card": card()}
    print(json.dumps(out), flush=True)
    names = [f"t{r:04d}" for r in range(1, args.nterms + 1)]
    tdict = tb.TermDictionary(names)
    texts = bench.gen_queries("and2", args.nq, args.nterms)[0] + bench.gen_queries("tree8", args.nq, args.nterms)[0] + phrases(args.nq, args.nterms)
    extra = workload(11_000, args.nterms, 0xADD)  # the added queries, shuffled
    rng = np.random.default_rng(0xC4)
    extra = [extra[i] for i in rng.permutation(len(extra))]
    cost = np.minimum(bench.synth_dfs(100_000_000, args.nterms), 0xFFFFFFFF).astype(np.uint32)
    w = 1.0 / np.arange(1, args.nterms + 1)
    w /= w.sum()
    docs = [rng.choice(args.nterms, size=args.doc_len, p=w).astype(np.uint32) for _ in range(args.ndocs)]
    parse = (lambda qs: [tb.parse_query(q, tdict) for q in qs])

    trees = parse(texts)  # parsing is the caller's, outside every timed call
    t0 = time.perf_counter()
    p = tb.Percolator(trees, nterms=args.nterms, term_cost=cost)
    reg_s = time.perf_counter() - t0
    res = {"queries": len(texts), "register_s": round(reg_s, 3), "registry_mb": round(p.info()["device_bytes"] / 1e6, 1)}
    live = list(range(len(texts)))
    steps, at = [], 0
    # the first add / remove of a process also loads the update kernels and allocates their scratch: one of each, reported apart
    for op, n in (("add", 1), ("remove", 1), ("add", 1), ("add", 1000), ("add", 30_000), ("remove", 1000), ("remove", 30_000)):
        if op == "add":
            batch = extra[at: at + n]
            at += n
            batch_trees = parse(batch)
            t0 = time.perf_counter()
            ids = p.add(batch_trees)
            host_ms = (time.perf_counter() - t0) * 1e3
            texts += batch
            live += ids.tolist()
        else:
            gone = rng.choice(len(live), n, replace=False)
            ids = np.array([live[i] for i in gone], np.uint32)
            t0 = time.perf_counter()
            p.remove(ids)
            host_ms = (time.perf_counter() - t0) * 1e3
            drop = set(gone.tolist())
            live = [q for i, q in enumerate(live) if i not in drop]
        t = p.last_update_timings()
        info = p.info()
        steps.append({"op": op + (" (first)" if len(steps) < 2 else ""), "n": n, "call_ms": round(host_ms, 3), "device_ms": round(t["device_ms"], 3), "live": info["nqueries"],
                      "next_id": info["next_id"], "anchor_entries": info["anchor_entries"], "registry_mb": round(info["device_bytes"] / 1e6, 1)})
        print(json.dumps(steps[-1]), flush=True)
    res["updates"] = steps

    live = sorted(live)
    live_trees = parse([texts[q] for q in live])
    t0 = time.perf_counter()
    fresh = tb.Percolator(live_trees, nterms=args.nterms, term_cost=cost)
    res["register_live_s"] = round(time.perf_counter() - t0, 3)
    p.percolate(docs)
    fresh.percolate(docs)  # warm-up
    runs = {"churned": [], "fresh": []}
    for _ in range(args.steps):
        for name, x in (("churned", p), ("fresh", fresh)):
            r = x.percolate(docs)
            runs[name].append((round(r.count_ms, 3), round(r.write_ms, 3), round(r.total_ms, 3)))
            if name == "churned":
                mine = r
            else:
                theirs = r
    lv = np.asarray(live, np.uint32)
    same = mine.candidates == theirs.candidates and all(np.array_equal(mine.document(d), lv[theirs.document(d)]) for d in range(args.ndocs))
    res["percolate_count_write_call_ms"] = runs
    res["churned_equals_fresh"] = bool(same)

    from percutil import RefPercolator
    nref = min(args.ref_docs, args.ndocs)
    ref = RefPercolator([(texts[q], 0, 0) for q in live], vocab=names)
    want = ref.run(docs[:nref])
    res["reference_parity"] = bool(all(np.array_equal(mine.document(d), lv[want[d]]) for d in range(nref)))
    out.update(churn=res)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
