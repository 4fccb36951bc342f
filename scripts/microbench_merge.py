"""Throughput of the segment merge (GpuIndexSource.merge_sources / trn_merge_sources): --gens generations indexed on the device, each of
--ndocs documents of --doc-len tokens drawn by Zipf(1) rank over --nterms terms (the indexer microbenchmark's documents), each replacing
--replace of the previous generation's documents; merged into one segment of each codec.  Reports the CUDA-event times of the decode,
merge (keep, rank, scatter) and encode kernels and of the assembly copy, the whole call's host time (uploads and copies included), the
postings read and written per second; `parity`: every file of the directory merged from the first --ref-gens generations equals the one the
reference's MergeCandidatesCollection::merge() writes (LUCENE index / hits.data: except the PFor padding the reference leaves
uninitialised), with the reference's time for that merge on one host thread.  One warm-up call, then the best of --steps calls.  The card
name, its power limit and SM clocks are read (not set) and printed.

--payloads P [P ...]: one set of generations per fraction P, in which a token carries a payload with probability P (sizes 1..8, random
bytes; P = 0: indexed without payloads), each merged through trn_merge_sources_payloads (P = 0: also through trn_merge_sources).  The
configurations' calls alternate, step after step, so that they share the card's state; one line per configuration.  The sources are
read from their directories and merged through one context; no source is uploaded for queries, so the merge has the card to itself.

    python scripts/microbench_merge.py [--gens 8] [--ndocs 2000000] [--doc-len 64] [--nterms 4096] [--replace 0.1] [--ref-gens 2] [--steps 3]
                                       [--payloads 0 0.3]
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
from idxutil import read_dir, term_names, zipf_corpus  # noqa: E402
from mergeutil import ref_merge  # noqa: E402
from trinity_b200.segments import SegmentCollection  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def same_dirs(got, want, codec):
    want, got = read_dir(want), read_dir(got)
    if sorted(want) != sorted(got):
        return False
    for f in want:
        if got[f].size != want[f].size:
            return False
        if codec == tb.CODEC_LUCENE and f in ("index", "hits.data"):
            if not np.all(got[f][got[f] != want[f]] == 0):
                return False
        elif not np.array_equal(got[f], want[f]):
            return False
    return True


def generations(g, root, args, frac):
    """--gens generations indexed on the device (codecs alternating); frac: the fraction of tokens with a payload (None: no payloads)"""
    step = int(args.ndocs * (1 - args.replace))
    paths, older = [], np.zeros(0, np.uint32)
    for k in range(args.gens):  # generation k: docIDs k*step+1 .. k*step+ndocs, the first ndocs - step of them replacing generation k-1's
        docids, offs, tok = zipf_corpus(args.ndocs, args.nterms, args.doc_len, 0xD0C5 + k)
        docids = docids + np.uint32(k * step)
        pay = ()
        if frac:
            rng = np.random.default_rng(0x9A7 + k)
            plens = np.where(rng.random(len(tok)) < frac, rng.integers(1, 9, len(tok)), 0).astype(np.uint8)
            pay = (None, plens, rng.integers(0, 1 << 63, size=len(tok), dtype=np.uint64) * np.uint64(2))
        p = Path(root) / f"{k + 1}"
        g.index_documents_flat(tb.CODEC_GOOGLE if k % 2 == 0 else tb.CODEC_LUCENE, docids, offs, tok, args.nterms, *pay).write(
            p, term_names(args.nterms), replaced=np.intersect1d(docids, older))
        older = docids
        paths.append(p)
    return paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gens", type=int, default=8)
    ap.add_argument("--ndocs", type=int, default=2_000_000)
    ap.add_argument("--doc-len", type=int, default=64)
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--replace", type=float, default=0.1)
    ap.add_argument("--ref-gens", type=int, default=2, help="generations of the prefix the reference merges and the files are compared on")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--payloads", type=float, nargs="+", default=None, help="fractions of tokens that carry a payload (see above)")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    g = tb.GpuIndexSource(0)
    with tempfile.TemporaryDirectory() as tmp:
        fracs = args.payloads if args.payloads is not None else [None]
        sets, configs = [], []  # sets: (paths oldest first, merge sources, segments); configs: (set, payload fraction, through trn_merge_sources_payloads)
        for i, f in enumerate(fracs):
            paths = generations(g, Path(tmp) / f"src{i}", args, f)
            segs = [tb.Segment(str(p)) for p in paths]  # alive while the sources point into them
            sets.append((paths, [tb.MergeSource.of_segment(s, str(p), int(p.name)) for s, p in zip(segs, paths)], segs))
            if f is None or f == 0:
                configs.append((i, f, False))
            if f is not None:
                configs.append((i, f, True))
        for codec, cname in ((tb.CODEC_GOOGLE, "google"), (tb.CODEC_LUCENE, "lucene")):
            for i, _, pay in configs:
                g.merge_sources(codec, sets[i][1], payloads=pay)  # warm-up
            runs = {c: [] for c in configs}
            for _ in range(args.steps):
                for c in configs:
                    runs[c].append(g.merge_sources(codec, sets[c[0]][1], payloads=c[2]))
            refs = {}
            for c in configs:
                i, f, pay = c
                best = min(runs[c], key=lambda r: r.timings["total_ms"])
                pr = lambda ms, n: round(n / (ms / 1e3), 0) if ms > 0 else None  # noqa: E731
                nread, nwritten = best.counts["postings_read"], best.counts["postings_written"]
                prefix = sets[i][0][:args.ref_gens]
                m = SegmentCollection(prefix).merge(codec, payloads=pay)
                m.write(Path(tmp) / f"dev_{cname}_{i}_{int(pay)}" / "100")
                if i not in refs:
                    refs[i] = ref_merge(codec, Path(tmp) / f"ref_{cname}_{i}" / "100", prefix, False, m.field_statistics["docsCnt"])[1]
                out = {"codec": cname, "gens": args.gens, "ndocs": args.ndocs, "doc_len": args.doc_len, "nterms": args.nterms,
                       "ms": {k: round(v, 3) for k, v in best.timings.items()}, "total_ms_all_runs": [round(r.timings["total_ms"], 1) for r in runs[c]],
                       "counts": best.counts, "postings_read_per_s": pr(best.timings["total_ms"], nread),
                       "postings_read_per_s_kernels": pr(best.timings["decode_ms"] + best.timings["merge_ms"] + best.timings["encode_ms"] + best.timings["assemble_ms"], nread),
                       "postings_written": nwritten, "index_bytes": int(best.index.size), "hits_bytes": int(best.hits.size),
                       "field_statistics": best.field_statistics,
                       "parity": same_dirs(Path(tmp) / f"dev_{cname}_{i}_{int(pay)}" / "100", Path(tmp) / f"ref_{cname}_{i}" / "100", codec), "ref_gens": args.ref_gens,
                       "ref_ms_one_thread": round(refs[i], 1), "device_ms_same_prefix": round(m.timings["total_ms"], 1)}
                if f is not None:
                    out["payloads"], out["entry"] = f, "trn_merge_sources_payloads" if pay else "trn_merge_sources"
                    out["decode_merge_encode_assemble_ms_all_runs"] = [[round(r.timings[k], 2) for k in ("decode_ms", "merge_ms", "encode_ms", "assemble_ms")] for r in runs[c]]
                print(json.dumps(out), flush=True)
    g.close()


if __name__ == "__main__":
    main()
