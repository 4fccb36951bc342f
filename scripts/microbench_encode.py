"""GPU-side encoders (trn_encode_google, trn_encode_lucene) vs the host encoder on the same postings: device time of the encode (kernels +
scans, without the host<->device copies), bytes identical.
Usage: python scripts/microbench_encode.py [ndocs] [first_rank] [nterms] [with_positions] [--codec google|lucene] [--whole-index]
--whole-index encodes every term of the synthetic index (4096 ranks) and compares with SynthIndex(codec, ndocs), the host encoder run over
the same postings on every core; otherwise the host encoder runs on one thread over the selected terms (default: the 16 densest)."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import trinity_b200 as tb  # noqa: E402

SYNTH_TERMS = 4096  # SynthIndex's default vocabulary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("ndocs", nargs="?", type=int, default=100_000_000)
    ap.add_argument("first_rank", nargs="?", type=int, default=1)
    ap.add_argument("nterms", nargs="?", type=int, default=16)
    ap.add_argument("with_positions", nargs="?", type=int, default=1)
    ap.add_argument("--codec", choices=["google", "lucene"], default="google")
    ap.add_argument("--whole-index", action="store_true", help=f"all {SYNTH_TERMS} terms, compared with SynthIndex")
    a = ap.parse_args()
    codec = tb.CODEC_LUCENE if a.codec == "lucene" else tb.CODEC_GOOGLE
    with_pos = a.with_positions != 0
    first, nterms = (1, SYNTH_TERMS) if a.whole_index else (a.first_rank, a.nterms)

    def term(rank):  # the ctypes calls release the GIL: the postings of many terms are generated at once
        d, f = tb.SynthIndex.postings(a.ndocs, rank, 1000, 0x5EED)
        p = tb.SynthIndex.positions(a.ndocs, rank, 1000, 0x5EED) if with_pos else None
        return d, f, p

    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        lists = list(ex.map(term, range(first, first + nterms)))
    posts = sum(len(l[0]) for l in lists)
    hits = sum(int(l[1].sum(dtype=np.uint64)) for l in lists)

    t0 = time.perf_counter()
    if a.whole_index:
        host = tb.SynthIndex(codec, a.ndocs, with_hits=with_pos)
        host_how = f"SynthIndex (generation + encode), {os.cpu_count()} threads"
        want_i, want_h, want_t = host.index, host.hits, host.terms
    else:
        b = tb.IndexBuilder(codec)
        for d, f, p in lists:
            b.add_term(d, f, p)
        host_how = "IndexBuilder, 1 thread"
        want_i, want_h, want_t = b.index(), b.hits(), b.terms_array()
    host_s = time.perf_counter() - t0

    g = tb.GpuIndexSource(0)
    best, hits_out = None, np.zeros(0, np.uint8)
    for _ in range(4):  # first call: allocations
        t0 = time.perf_counter()
        if codec == tb.CODEC_LUCENE:
            index, hits_out, terms, ms = g.encode_lucene(lists)
        else:
            index, terms, _, ms = g.encode_google(lists)
        wall = time.perf_counter() - t0
        best = ms if best is None else min(best, ms)
    same = bool(index.size == want_i.size and np.array_equal(index, want_i) and np.array_equal(terms, want_t))
    if codec == tb.CODEC_LUCENE:
        same = same and bool(hits_out.size == want_h.size and np.array_equal(hits_out, want_h))
    # docids + freqs (+ positions) + the hit offsets (the LUCENE encoder always scans the freqs: its hit blocks cross documents)
    in_bytes = posts * 8 + (hits * 4 if with_pos else 0) + (posts * 8 if with_pos or codec == tb.CODEC_LUCENE else 0)
    out_bytes = int(index.size) + int(hits_out.size)
    host_key = "host_encoder_s_all_threads" if a.whole_index else "host_encoder_s_1_thread"
    print(json.dumps({"what": f"{a.codec.upper()} encode, device vs host", "ndocs": a.ndocs, "terms": [first, first + nterms - 1], "postings": posts,
                      "hits": hits, "with_positions": with_pos, "index_bytes": int(index.size), "hits_bytes": int(hits_out.size),
                      "bytes_identical_to_host_encoder": same, "device_ms": round(best, 3), "postings_per_s_device": posts / (best / 1e3),
                      "in_plus_out_GBps": (in_bytes + out_bytes) / (best / 1e3) / 1e9, "call_wall_s_incl_copies": round(wall, 3),
                      "host_encoder": host_how, host_key: round(host_s, 3), "host_postings_per_s": posts / host_s}))
    assert same


if __name__ == "__main__":
    main()
