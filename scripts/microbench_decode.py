#!/usr/bin/env python
"""configs[4]: postings-decode microbench — whole-list decode of every term of the synthetic index, materialised (8 B/posting written)
and fused (checksum only), both codecs, vs the HBM roofline.  usage: microbench_decode.py [ndocs] [filter e.g. google-fused]
Every run checks the per-term sums of docIDs and freqs against the generator's closed form for a few terms."""
import json, sys, time
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import trinity_b200 as tb

ndocs = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
only = sys.argv[2].lower() if len(sys.argv) > 2 else ""
peak = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 3350.0  # H100 SXM data sheet
for codec, name in ((0, "GOOGLE"), (1, "LUCENE")):
    if only and not only.startswith(name.lower()):
        continue
    s = tb.SynthIndex(codec, ndocs, 4096)
    g = tb.GpuIndexSource(0)
    g.upload(codec, np.asarray(s.index), np.asarray(s.terms), ndocs)
    terms = list(range(4096))
    postings = int(s.terms["documents"].sum())
    chunk_bytes = int(s.terms["chunk_len"].sum())
    want = {}
    for t in (4095, 2000, 300):
        d, f = tb.SynthIndex.postings(ndocs, t + 1)
        want[t] = (int(d.astype(np.uint64).sum()), int(f.astype(np.uint64).sum()))
    for mat in (False, True):
        variant = "materialised" if mat else "fused-checksum"
        if only and "-" in only and not variant.startswith(only.split("-", 1)[1]):
            continue
        if mat and postings * 8 > 20e9:
            continue
        best = 1e9
        for it in range(5):
            # materialised variant: only the kernel is timed (device_ms); the D2H of 8 B/posting is outside the event pair
            d, f, sums, ms = g.decode_terms(terms, materialise=mat)
            if it >= 2:
                best = min(best, ms)
        ok = all(int(sums[t, 0]) == want[t][0] and int(sums[t, 1]) == want[t][1] for t in want)
        algo = chunk_bytes + (8 * postings if mat else 0)
        print(json.dumps({"codec": name, "variant": variant, "ndocs": ndocs, "postings": postings, "kernel_ms": best, "postings_per_s": postings / (best * 1e-3),
                          "algorithmic_bytes": algo, "achieved_gbs": algo / (best * 1e-3) / 1e9, "peak_gbs": peak, "frac": algo / (best * 1e-3) / 1e9 / peak,
                          "bytes_per_posting": chunk_bytes / postings, "checksums_ok": ok}), flush=True)
    g.close()
