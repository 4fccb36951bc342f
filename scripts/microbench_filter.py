"""Cost of per-query document filters (trn_exec_batch_filtered) on bench.py's batches at bench.py's size: and2, tree8 and and2l
(DocumentsOnly) and or10 (BM25 top-100), each run unfiltered and with per-query allow sets of density 1e-4, 1e-2 and 0.5 and deny sets of
density 1e-2 and 0.5, the arms alternating step by step.  The queries of a batch take their set round-robin from a pool of --pool
random sets of that density.

Reported per batch and arm: the best and median host time of the whole call (plans in, results in host memory), the exec kernels' device
time (trn_timings.kernel_ms).  Parity, on --sample queries spread over the batch: a DocumentsOnly arm's documents equal
the unfiltered run's documents restricted on the host (bench.py checks the unfiltered batch against the reference), and match_counts
equal their number; a top-k arm's documents all pass the filter, its match_counts equal the unfiltered SCORED_ALL run restricted on the
host, and its scores equal that run's restricted top-k scores (rtol 1e-5).  The card name and its power limit are printed with the numbers (read-only nvidia-smi query).

    python scripts/microbench_filter.py [--nq 1000] [--steps 5] [--pool 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
import trinity_b200 as tb  # noqa: E402

ARMS = [("allow", 1e-4), ("allow", 1e-2), ("allow", 0.5), ("deny", 1e-2), ("deny", 0.5)]
BATCHES = [("and2", tb.CODEC_GOOGLE, tb.MODE_DOCS_ONLY), ("tree8", tb.CODEC_GOOGLE, tb.MODE_DOCS_ONLY), ("and2l", tb.CODEC_LUCENE, tb.MODE_DOCS_ONLY),
           ("or10", tb.CODEC_LUCENE, tb.MODE_SCORED_TOPK)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def random_set(rng, ndocs, density):
    if density >= 0.1:
        return np.flatnonzero(rng.random(ndocs, dtype=np.float32) < density).astype(np.uint32) + 1
    return np.unique(rng.integers(1, ndocs + 1, int(ndocs * density), dtype=np.uint32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ndocs", type=int, default=100_000_000)
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool", type=int, default=4, help="distinct sets per density (queries share them round-robin)")
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--sample", type=int, default=8, help="queries of every batch checked for parity")
    args = ap.parse_args()
    out = {"card": card(), "ndocs": args.ndocs, "nq": args.nq, "steps": args.steps}
    print(json.dumps({"card": out["card"]}), flush=True)
    rng = np.random.default_rng(0xF11)
    pools = {arm: [random_set(rng, args.ndocs, arm[1]) for _ in range(args.pool)] for arm in ARMS}
    threads = max(1, len(os.sched_getaffinity(0)))
    cache = {}

    def members(arm, i):
        """membership of every docID in pool set i of the arm (built once)"""
        if (arm, i) not in cache:
            b = np.zeros(args.ndocs + 1, bool)
            b[pools[arm][i]] = True
            cache[(arm, i)] = b
        return cache[(arm, i)]

    for codec in (tb.CODEC_GOOGLE, tb.CODEC_LUCENE):
        synth = tb.SynthIndex(codec, args.ndocs, args.nterms, threads=threads)
        g = tb.GpuIndexSource(0)
        g.upload(codec, np.asarray(synth.index), np.asarray(synth.terms), args.ndocs)
        tdict = tb.TermDictionary(synth.names)
        sets = {arm: [g.docset(s) for s in pools[arm]] for arm in ARMS}
        for wl, wcodec, mode in BATCHES:
            if wcodec != codec:
                continue
            texts, _ = bench.gen_queries(wl, args.nq, args.nterms)
            scored = mode != tb.MODE_DOCS_ONLY
            plans = [tb.parse_query(t, tdict) for t in texts]
            if scored:
                plans = [g.set_bm25_weights(p, args.ndocs) for p in plans]
            packed = g.pack(plans)
            filters = {None: None}
            for arm in ARMS:
                side = arm[0]
                filters[arm] = [tb.DocFilter(allow=sets[arm][q % args.pool]) if side == "allow" else tb.DocFilter(deny=sets[arm][q % args.pool])
                                for q in range(len(plans))]
            # parity on a sample of the batch's queries
            sample = list(range(0, len(plans), max(1, len(plans) // args.sample)))[: args.sample]
            splans = [plans[q] for q in sample]
            base = g.exec_batch(splans, tb.MODE_SCORED_ALL if scored else mode, k=args.k)
            res = {"queries": len(plans), "mode": "top-%d" % args.k if scored else "docs", "parity_queries": len(sample)}
            for arm in ARMS:
                r = g.exec_batch(splans, mode, k=args.k, filters=[filters[arm][q] for q in sample])
                ok = True
                for i, q in enumerate(sample):
                    member = members(arm, q % args.pool)
                    bd, bs = base.query(i)
                    m = member[bd] if arm[0] == "allow" else ~member[bd]
                    gd, gs = r.query(i)
                    ok &= int(r.match_counts[i]) == int(m.sum())
                    if scored:
                        want = np.sort(bs[m])[::-1][: args.k]
                        gm = member[gd] if arm[0] == "allow" else ~member[gd]
                        ok &= bool(np.all(gm)) and len(gs) == len(want) and bool(np.allclose(gs, want, rtol=1e-5, atol=0))
                    else:
                        ok &= np.array_equal(gd, bd[m])
                res[f"{arm[0]}-{arm[1]:g}"] = {"parity": bool(ok)}
            # timing: the arms alternate step by step
            keys = [None] + ARMS
            times = {a: [] for a in keys}
            kms = {a: [] for a in keys}
            for step in range(args.warmup + args.steps):
                for a in keys:
                    t0 = time.perf_counter()
                    g.exec_batch(plans, mode, k=args.k, copy=False, packed=packed, filters=filters[a])
                    t1 = time.perf_counter()
                    if step >= args.warmup:
                        times[a].append((t1 - t0) * 1e3)
                        kms[a].append(g.last_timings()["kernel_ms"])
            for a in keys:
                name = "unfiltered" if a is None else f"{a[0]}-{a[1]:g}"
                res.setdefault(name, {}).update({"call_ms_best": round(min(times[a]), 3), "call_ms_median": round(float(np.median(times[a])), 3),
                                                 "kernel_ms_median": round(float(np.median(kms[a])), 3)})
            out[wl] = res
            print(json.dumps({wl: res}), flush=True)
        for arm in ARMS:
            for s in sets[arm]:
                s.close()
        g.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
