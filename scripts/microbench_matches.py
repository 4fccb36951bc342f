"""Throughput of the default exec mode (GpuIndexSource.exec_matches) on bench.py's 100M-document GOOGLE index: for a prefix of the and2,
tree8 and or10 batches, matches/s, matched terms/s and hits/s, with the device time of the docs pass, of the count kernel with its scans,
and of the write kernel (CUDA events around the kernels alone; the whole call's time, copies and host synchronisations included, beside
them).

Checks: the docIDs equal the same queries in DocumentsOnly mode (queries with a root filter over a disjunction are left out: there the
reference's DocumentsOnly quirk keeps what this mode excludes); every match holds a term and every term as many hits as its freq; and for
--sample matches spread over the result, every matched term's freq, positions, payload lengths and payloads equal trn_debug_hits, the
same hit walker run on the host over the index bytes (tests/test_matched_terms_cpu pins it against the reference's materialize_hits).
The card name and its power limit are printed with the numbers (read-only nvidia-smi query).

    python scripts/microbench_matches.py [--nq 20] [--nq-or10 2] [--steps 3] [--sample 300]
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
import trinity_b200 as tb  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        return out
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def root_filter_over_or(nodes):
    cur = 0
    while nodes[cur]["kind"] == tb.NODE_NOT:
        cur = int(nodes[cur]["first_child"])
    return cur != 0 and nodes[cur]["kind"] == tb.NODE_OR


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ndocs", type=int, default=100_000_000)
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=20, help="queries of the and2 and tree8 prefixes (the full batches return hundreds of GB of hits)")
    ap.add_argument("--nq-or10", type=int, default=2, help="queries of the or10 prefix (each matches ~10 %% of the documents)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=300, help="matches per batch whose hits are checked against trn_debug_hits")
    args = ap.parse_args()
    synth = tb.SynthIndex(tb.CODEC_GOOGLE, args.ndocs, args.nterms, threads=max(1, len(os.sched_getaffinity(0))))
    g = tb.GpuIndexSource(0)
    g.upload(tb.CODEC_GOOGLE, np.asarray(synth.index), np.asarray(synth.terms), args.ndocs)
    tdict = tb.TermDictionary(synth.names)
    out = {"card": card(), "ndocs": args.ndocs, "nq": args.nq}
    print(json.dumps({"card": out["card"]}), flush=True)
    for wl in ("and2", "tree8", "or10"):
        texts, _ = bench.gen_queries(wl, args.nq_or10 if wl == "or10" else args.nq, args.nterms)
        plans = [tb.parse_query(t, tdict) for t in texts]
        res = g.exec_matches(plans)  # warm-up, and the result checked below
        docs = g.exec_batch(plans, tb.MODE_DOCS_ONLY)
        # a root filter over a disjunction excludes in this mode and not in DocumentsOnly (the reference quirk): those are left out
        plain = [q for q, p in enumerate(plans) if not root_filter_over_or(p)]
        parity = all(np.array_equal(res.query(q), docs.query(q)[0]) for q in plain)
        parity &= bool(np.all(np.diff(res.term_offsets) >= 1)) and bool(np.all(np.diff(res.hit_offsets) == res.freqs))
        rng = np.random.default_rng(7)
        index, terms = np.asarray(synth.index), np.asarray(synth.terms)
        sampled = rng.choice(len(res.docids), size=min(args.sample, len(res.docids)), replace=False) if len(res.docids) else []
        by_term = {}  # term -> [(docID, position in res.terms)]: one host directory build per term
        for m in sampled:
            for t in range(int(res.term_offsets[m]), int(res.term_offsets[m + 1])):
                by_term.setdefault(int(res.terms[t]), []).append((int(res.docids[m]), t))
        for term, pairs in by_term.items():
            got = tb.debug_hits(tb.CODEC_GOOGLE, index, None, terms[term], [d for d, _ in pairs])
            for want, (_, t) in zip(got, pairs):
                h = res.hits[int(res.hit_offsets[t]): int(res.hit_offsets[t + 1])]
                parity &= want is not None and want[0] == int(res.freqs[t]) and np.array_equal(want[1], h["pos"]) \
                    and np.array_equal(want[2], h["payload_len"]) and np.array_equal(want[3], h["payload"])
        best = None
        for _ in range(args.steps):
            r = g.exec_matches(plans)
            if best is None or r.device_ms < best.device_ms:
                best = r
        m, t, h = len(best.docids), len(best.terms), len(best.hits)
        s = best.device_ms / 1e3
        k = (best.docs_ms + best.count_ms + best.write_ms) / 1e3  # the kernels alone
        out[wl] = {"queries": len(plans), "matches": m, "terms": t, "hits": h, "call_ms": round(best.device_ms, 3), "docs_pass_ms": round(best.docs_ms, 3),
                   "count_ms": round(best.count_ms, 3), "write_ms": round(best.write_ms, 3), "matches_per_s": round(m / k), "terms_per_s": round(t / k),
                   "hits_per_s": round(h / k), "matches_per_s_call": round(m / s), "chunks": best.chunks, "parity": bool(parity),
                   "docs_only_queries": len(plain), "sampled_matches": len(sampled)}
        print(json.dumps({wl: out[wl]}), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
