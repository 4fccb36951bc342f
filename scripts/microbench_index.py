"""Throughput of the indexer (GpuIndexSource.index_documents / trn_index_documents): documents of tokens drawn by Zipf(1) rank over a
4096-term vocabulary (the percolator microbenchmark's documents), 64 tokens each, both codecs.  Reports tokens/s of the sort (document
ranks, keys, radix passes), the postings pass and the encoder from the CUDA events of the kernels alone, and of the whole call (host time,
copies included); the radix passes run; the output sizes; `parity`: every file of the directory written from a --ref-ndocs prefix equals the
one the reference's SegmentIndexSession::commit() writes for that prefix (LUCENE index / hits.data: except the PFor padding the reference
leaves uninitialised); and the reference's time for that prefix on one host thread (oracle/_ref/libtrinity_ref_indexer.so).  One warm-up
call, then the best of --steps calls with the spread.  The card name, its power limit and SM clocks are read (not set) and printed.

--payloads: every token also carries a random payload of 0..8 bytes (trn_index_documents_payloads); each codec then runs the batch
without and with payloads alternately, --steps calls of each, and prints one line per variant (the payload line's parity is against the
reference fed the same payloads).

4 M documents x 64 tokens are 2.6e8 keys: two key buffers, the flags and their scans take about 11 GB of HBM beside the 2 GB of inputs.

    python scripts/microbench_index.py [--ndocs 4000000] [--doc-len 64] [--nterms 4096] [--ref-ndocs 200000] [--steps 3] [--payloads]
"""
import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import trinity_b200 as tb  # noqa: E402
from idxutil import read_dir, ref_index_flat, term_names, zipf_corpus  # noqa: E402
from payutil import ref_index_payloads, zipf_payloads  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def parity(g, codec, names, docids, offs, tok, n, length, pay=None):
    d, o, t = docids[:n], offs[:n + 1], tok[:n * length]
    with tempfile.TemporaryDirectory() as tmp:
        if pay is None:
            ref_ms = ref_index_flat(codec, Path(tmp) / "r" / "1", names, d, o, t)
            g.index_documents_flat(codec, d, o, t, len(names)).write(Path(tmp) / "w" / "1", names)
        else:
            pl, pv = pay[0][:n * length], pay[1][:n * length]
            ref_ms = ref_index_payloads(codec, Path(tmp) / "r" / "1", names, d, o, t, None, pl, pv)
            g.index_documents_flat(codec, d, o, t, len(names), None, pl, pv).write(Path(tmp) / "w" / "1", names)
        want, got = read_dir(Path(tmp) / "r" / "1"), read_dir(Path(tmp) / "w" / "1")
    same = sorted(want) == sorted(got)
    for f in want:
        if not same:
            break
        if got[f].size != want[f].size:
            same = False
        elif codec == tb.CODEC_LUCENE and f in ("index", "hits.data"):
            same = bool(np.all(got[f][got[f] != want[f]] == 0))
        else:
            same = bool(np.array_equal(got[f], want[f]))
    return same, ref_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ndocs", type=int, default=4_000_000)
    ap.add_argument("--doc-len", type=int, default=64)
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--ref-ndocs", type=int, default=200_000, help="documents of the prefix the reference indexes and the files are compared on")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--payloads", action="store_true", help="also index every token with a payload, alternating with the payload-free calls")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    names = term_names(args.nterms)
    docids, offs, tok = zipf_corpus(args.ndocs, args.nterms, args.doc_len, 0xD0C5)
    ntok = len(tok)
    pay = zipf_payloads(np.random.default_rng(0xFA7), ntok) if args.payloads else None
    variants = [None, pay] if args.payloads else [None]
    g = tb.GpuIndexSource(0)
    for codec, cname in ((tb.CODEC_GOOGLE, "google"), (tb.CODEC_LUCENE, "lucene")):
        call = lambda p: g.index_documents_flat(codec, docids, offs, tok, args.nterms, None, *(p if p is not None else (None, None)))  # noqa: E731
        for p in variants:
            call(p)  # warm-up: module load, first allocations
        allruns = [[] for _ in variants]
        for _ in range(args.steps):  # the variants alternate, so drift of the card's clocks touches both alike
            for v, p in enumerate(variants):
                allruns[v].append(call(p))
        for p, runs in zip(variants, allruns):
            report(g, args, codec, cname, names, docids, offs, tok, ntok, p, runs)
    g.close()


def report(g, args, codec, cname, names, docids, offs, tok, ntok, pay, runs):
    best = min(runs, key=lambda r: r.timings["total_ms"])
    rate = lambda ms: round(ntok / (ms / 1e3), 0) if ms > 0 else None  # noqa: E731
    nref = min(args.ref_ndocs, args.ndocs)
    same, ref_ms = parity(g, codec, names, docids, offs, tok, nref, args.doc_len, pay)
    out = {"codec": cname, "payloads": pay is not None, "ndocs": args.ndocs, "tokens": ntok, "nterms": args.nterms, "sort_passes": best.sort_passes,
           "passes_skipped": 16 - best.sort_passes,  # of the 8 + 8 byte-wide passes of two full 64-bit sorts
           "ms": {k: round(v, 3) for k, v in best.timings.items()},
           "total_ms_all_runs": [round(r.timings["total_ms"], 1) for r in runs],
           "tokens_per_s": {k[:-3]: rate(v) for k, v in best.timings.items()},
           "index_bytes": int(best.index.size), "hits_bytes": int(best.hits.size), "postings": best.field_statistics["sumTermsDocs"],
           "parity": same, "ref_ndocs": nref, "ref_ms_one_thread": round(ref_ms, 1), "ref_tokens_per_s": round(nref * args.doc_len / (ref_ms / 1e3), 0)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
