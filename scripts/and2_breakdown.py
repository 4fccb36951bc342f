"""Time the and2 batch of bench.py by route class: with the flat ANDs on their run-major tickets (the default), with TRN_MIXED_RUNS=0 (the
flat ANDs with one bitmap operand on per-tile tickets) and with TRN_DENSE_RUNS=0 TRN_MIXED_RUNS=0 (every flat AND on per-tile tickets).

Builds bench.py's GOOGLE index and and2 batch, splits the batch into
  both    flat AND, both operands with a resident bitmap
  one     flat AND, one operand with a bitmap
  none    flat AND, no bitmap
  cand    candidate-driven
and times each class as its own device-resident batch (exec_batch_device, as bench.py; CUDA events over --steps steps after --warmup) on
three sources over the same index, created with those settings, alternating.  Per class it prints ms per step, (query, tile) work
items (candidate-driven: lead-term groups), matches, result words, and the modelled HBM bytes of bitmap reads: per-tile order (every
item reads its operands' tile words) and run-major order (every bitmap run read once).  Needs a GPU; prints the card and its power limit.

    python scripts/and2_breakdown.py [--ndocs 100000000] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
import trinity_b200 as tb  # noqa: E402


SETTINGS = {"runs": {}, "mixed_tiles": {"TRN_MIXED_RUNS": "0"}, "tiles": {"TRN_DENSE_RUNS": "0", "TRN_MIXED_RUNS": "0"}}


def source(synth, ndocs, env):
    os.environ.update(env)
    try:
        g = tb.GpuIndexSource(0)
    finally:
        for k in env:
            os.environ.pop(k)
    g.upload(tb.CODEC_GOOGLE, np.asarray(synth.index), np.asarray(synth.terms), ndocs)
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ndocs", type=int, default=100_000_000)
    ap.add_argument("--nterms", type=int, default=4096)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two sources per class")
    args = ap.parse_args()
    import torch

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    synth = tb.SynthIndex(tb.CODEC_GOOGLE, args.ndocs, args.nterms, threads=max(1, len(os.sched_getaffinity(0))))
    srcs = {k: source(synth, args.ndocs, env) for k, env in SETTINGS.items()}
    g = srcs["runs"]
    texts, _ = bench.gen_queries("and2", args.nq, args.nterms)
    tdict = tb.TermDictionary(synth.names)
    plans = [tb.parse_query(q, tdict) for q in texts]
    terms = np.asarray(synth.terms)
    g.exec_batch(plans, tb.MODE_DOCS_COMPACT, copy=False)
    routes = g.last_routes()
    dense = {}  # term -> bitmap bytes

    def bitmap_bytes(t):
        if t not in dense:
            bm = g.dense_bitmap(t)
            dense[t] = 0 if bm is None else len(bm[1]) * 4
        return dense[t]

    tile = 1 << 14
    tiles = (args.ndocs >> 14) + 1  # the synthetic terms spread over the whole docID range
    classes = {"both": [], "one": [], "none": [], "cand": []}
    for i, p in enumerate(plans):
        ts = [int(x["term"]) for x in p if x["kind"] == tb.NODE_TERM]
        nd = sum(bitmap_bytes(t) > 0 for t in ts)
        if routes[i] == tb.ROUTE_CANDIDATE:
            classes["cand"].append(i)
        elif routes[i] == tb.ROUTE_FLAT_AND:
            classes["both" if nd == len(ts) else "one" if nd else "none"].append(i)
    print(json.dumps({"card": card, "ndocs": args.ndocs, "nq": args.nq, "dense_terms": g.info()["dense_terms"],
                      "dense_bitmap_bytes": g.info()["dense_bitmap_bytes"]}))
    stream = torch.cuda.current_stream()
    for name, qs in classes.items():
        if not qs:
            continue
        sub = [plans[i] for i in qs]
        items = old_b = 0
        used = set()
        for i in qs:
            ts = [int(x["term"]) for x in plans[i] if x["kind"] == tb.NODE_TERM]
            if name == "cand":  # 32-block groups of the lead (rarest) term
                lead_blocks = -(-min(int(terms["documents"][t]) for t in ts) // 32)
                items += -(-lead_blocks // 32)
            else:
                items += tiles
                nd = [t for t in ts if bitmap_bytes(t)]
                old_b += tiles * len(nd) * (tile // 8)
                used |= set(nd)
        # run-major order reads each bitmap the class uses once; the other classes keep the per-tile order
        new_b = sum(bitmap_bytes(t) for t in used) if name in ("both", "one") else old_b
        ms = {k: [] for k in srcs}
        for _ in range(args.rounds):
            for key, s in srcs.items():
                packed = s.pack(sub)
                for _ in range(args.warmup):
                    s.exec_batch_device(sub, tb.MODE_DOCS_COMPACT, packed=packed)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.steps):
                    s.exec_batch_device(sub, tb.MODE_DOCS_COMPACT, packed=packed)
                e1.record(stream)
                torch.cuda.synchronize()
                ms[key].append(e0.elapsed_time(e1) / args.steps)
        res = g.exec_batch(sub, tb.MODE_DOCS_COMPACT, copy=False)
        print(json.dumps({"class": name, "queries": len(qs), "work_items": items, "matches": int(res.match_counts.sum()),
                          "result_bytes": res.result_bytes(), **{f"ms_per_step_{k}": [round(x, 3) for x in v] for k, v in ms.items()},
                          "bitmap_bytes_per_tile_order": old_b,
                          "bitmap_bytes_run_major": new_b}))
    for s in srcs.values():
        s.close()


if __name__ == "__main__":
    main()
