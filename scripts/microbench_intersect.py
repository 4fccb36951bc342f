"""Throughput of the query-token intersections (GpuIndexSource.intersect_batch / trn_intersect) on bench.py's 100M-document index, both
codecs: requests are the term sets of bench.py's and2 (2 groups) and tree8 (8 groups) batches, one term per group.  Reports the device
time of pass A and of pass B (CUDA events around the kernels alone), the host time of the epoch planner, the whole call's time,
postings/s and requests/s; then runs the reference's own intersect() (oracle/_ref/libtrinity_ref_isect.so, one host thread) over a
prefix of the requests on the same index bytes and compares every result of that prefix as a {mask: count} dict.  The card name and
its power limit are printed with the numbers (read-only nvidia-smi query).

    python scripts/microbench_intersect.py [--nq 200] [--ref-nq 4] [--steps 3] [--codecs google,lucene]
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
sys.path.insert(0, str(ROOT / "tests"))

import bench  # noqa: E402
import trinity_b200 as tb  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ndocs", type=int, default=100_000_000)
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=200, help="requests per batch (and2 and tree8 term sets)")
    ap.add_argument("--ref-nq", type=int, default=4, help="requests of each batch's prefix run through the reference and compared")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--codecs", default="google,lucene")
    args = ap.parse_args()
    from isectutil import RefIsect
    risect = RefIsect()
    out = {"card": card(), "ndocs": args.ndocs, "nq": args.nq}
    print(json.dumps({"card": out["card"]}), flush=True)
    for cname in args.codecs.split(","):
        codec = tb.CODEC_GOOGLE if cname == "google" else tb.CODEC_LUCENE
        synth = tb.SynthIndex(codec, args.ndocs, args.nterms, threads=max(1, len(os.sched_getaffinity(0))))
        index, terms = np.asarray(synth.index), np.asarray(synth.terms)
        hits = np.asarray(synth.hits) if codec == tb.CODEC_LUCENE else None
        g = tb.GpuIndexSource(0)
        g.upload(codec, index, terms, args.ndocs)
        ref = risect.source(codec, index, synth.names, terms, hits)
        for wl in ("and2", "tree8"):
            _, ranks = bench.gen_queries(wl, args.nq, args.nterms)
            reqs = [[[int(t)] for t in r] for r in ranks]
            g.intersect_batch(reqs)  # warm-up
            best = None
            for _ in range(args.steps):
                r = g.intersect_batch(reqs)
                if best is None or r.total_ms < best.total_ms:
                    best = r
            kern = (best.masks_ms + best.count_ms) / 1e3
            parity, ref_s = True, 0.0
            for i in range(min(args.ref_nq, len(reqs))):
                t0 = time.perf_counter()
                want = ref.intersect([[synth.names[t] for t in grp] for grp in reqs[i]])
                ref_s += time.perf_counter() - t0
                parity &= dict(want) == dict(best[i])
            nref = min(args.ref_nq, len(reqs))
            res = {"requests": len(reqs), "postings": best.postings, "distinct_masks": best.distinct, "pass_a_ms": round(best.masks_ms, 3),
                   "plan_ms": round(best.plan_ms, 3), "pass_b_ms": round(best.count_ms, 3), "call_ms": round(best.total_ms, 3),
                   "postings_per_s_kernels": round(best.postings / kern) if kern else None, "requests_per_s_call": round(len(reqs) / (best.total_ms / 1e3)),
                   "reference_requests": nref, "reference_s_per_request_1_thread": round(ref_s / max(1, nref), 3),
                   "parity": bool(parity)}
            ref_post = sum(int(terms["documents"][t]) for req in reqs[:nref] for grp in req for t in grp)
            res["reference_postings_per_s_1_thread"] = round(ref_post / ref_s) if ref_s else None
            out[f"{wl}_{cname}"] = res
            print(json.dumps({f"{wl}_{cname}": res}), flush=True)
        del g, ref, synth
    print(json.dumps(out))


if __name__ == "__main__":
    main()
