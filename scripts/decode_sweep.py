#!/usr/bin/env python
"""BASELINE.json configs[4]: postings-decode microbench — block-size / skip-list sweep vs the HBM roofline.

The GOOGLE layout's two compile-time constants (google_codec.h:17-20: N = 32 documents per block, SKIPLIST_STEP = 8 blocks per skiplist
entry) are varied at index-build time (trn_synth_build_ex), with and without inline positions; LUCENE's block size is fixed at 128 by
its FastPFor page (lucene_codec.h:48-57: the 64-value alternative is compiled out in the reference), so it appears as one point.
Every point decodes EVERY posting of the 100M-document synthetic index (k_decode_stream_*: bulk-copy staging, checksums compared with the
generator's closed form) and reports kernel time, postings/s and achieved bytes/s of the term chunks against the measured HBM peak.

With --device-encode the GOOGLE points are ENCODED ON THE GPU (trn_encode_google, the device-side Encoder of SURVEY.md 8(f) row 4): the postings
are generated once, every geometry is one device encode of the whole index — no CPU re-encode per point.

usage: decode_sweep.py [ndocs] [out.json] [--device-encode]"""
import json, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import trinity_b200 as tb

import time
device_encode = "--device-encode" in sys.argv
argv = [a for a in sys.argv if a != "--device-encode"]
ndocs = int(argv[1]) if len(argv) > 1 else 100_000_000
out_path = argv[2] if len(argv) > 2 else None
peak = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 3350.0  # H100 SXM data sheet
NT = 4096
want = {}
for t in (4095, 2000, 300):
    d, f = tb.SynthIndex.postings(ndocs, t + 1)
    want[t] = (int(d.astype(np.uint64).sum()), int(f.astype(np.uint64).sum()))

lists = None
if device_encode:  # the postings of every term, once (document order; positions as the synthetic generator places them)
    t0 = time.time()
    lists = []
    for r in range(1, NT + 1):
        d, f = tb.SynthIndex.postings(ndocs, r)
        lists.append((d, f, tb.SynthIndex.positions(ndocs, r)))
    print(f"postings generated in {time.time() - t0:.1f} s", flush=True)

points = []
grid = [(0, bd, 8, True) for bd in (8, 16, 32, 64, 128)] + [(0, 32, st, True) for st in (1, 64)] + [(0, bd, 8, False) for bd in (16, 32, 64)] + [(1, 128, 1, True)]
if device_encode:  # the GOOGLE geometries with positions: five device encodes of the whole index
    grid = [(0, bd, 8, True) for bd in (16, 32, 64)] + [(0, 32, st, True) for st in (1, 64)]
for codec, bd, step, hits in grid:
    g = tb.GpuIndexSource(0)
    enc = None
    if device_encode and codec == 0:
        t0 = time.time()
        index, tarr, _, enc_ms = g.encode_google(lists if hits else [(d, f, None) for d, f, _ in lists], bd, step)
        enc = {"encoded_on": "device (trn_encode_google)", "device_ms": enc_ms, "call_s_incl_copies": time.time() - t0}
        s = None
    else:
        s = tb.SynthIndex(codec, ndocs, NT, with_hits=hits, google_block_docs=bd, google_skiplist_step=step)
        index, tarr = np.asarray(s.index), np.asarray(s.terms)
    g.upload(codec, index, tarr, ndocs)
    postings = int(tarr["documents"].sum())
    chunk_bytes = int(tarr["chunk_len"].sum())
    terms = list(range(NT))
    row = {"codec": "GOOGLE" if codec == 0 else "LUCENE", "block_docs": bd, "skiplist_step": step, "positions": hits, "ndocs": ndocs, "postings": postings,
           "chunk_bytes": chunk_bytes, "bytes_per_posting": chunk_bytes / postings, "detected_block_docs": g.info()["block_docs"]}
    if enc:
        row["encode"] = enc
    for mat in (False, True):
        best = 1e9
        for it in range(5):
            _, _, sums, ms = g.decode_terms(terms, materialise=mat)
            if it >= 2:
                best = min(best, ms)
        ok = all(int(sums[t, 0]) == want[t][0] and int(sums[t, 1]) == want[t][1] for t in want)
        algo = chunk_bytes + (8 * postings if mat else 0)
        key = "materialised" if mat else "fused"
        row[key] = {"kernel_ms": best, "postings_per_s": postings / (best * 1e-3), "algorithmic_bytes": algo, "achieved_gbs": algo / (best * 1e-3) / 1e9,
                    "frac_of_measured_hbm_peak": algo / (best * 1e-3) / 1e9 / peak, "checksums_ok": ok}
    points.append(row)
    print(json.dumps(row), flush=True)
    g.close()
    del s
best = max((p for p in points if p["codec"] == "GOOGLE"), key=lambda p: p["fused"]["frac_of_measured_hbm_peak"])
summary = {"peak_gbs": peak, "peak_source": "MEASURED_PEAKS.json hbm_gbs" if (ROOT / "MEASURED_PEAKS.json").exists() else "fallback", "points": points,
           "best_google_fused": {k: best[k] for k in ("block_docs", "skiplist_step", "positions")} | best["fused"]}
if out_path:
    Path(out_path).write_text(json.dumps(summary, indent=1))
print("BEST", json.dumps(summary["best_google_fused"]))
