"""Time the and2 batch of bench.py by route class, on sources created with different settings, alternating: the default (every run-major
ticket space on, both tiers of resident bitmaps), TRN_PROBE_BITMAPS=0 (no probe bitmaps: the candidate-driven conjunction probes every
term without a dense bitmap through its block directory), TRN_CAND_RUNS=0 (candidate-driven groups in query order), and on request TRN_MIXED_RUNS=0 (the flat ANDs with one
bitmap operand on per-tile tickets) and TRN_DENSE_RUNS=0 TRN_MIXED_RUNS=0 (every flat AND on per-tile tickets).

Builds bench.py's GOOGLE index and and2 batch, splits the batch into
  both        flat AND, both operands with a resident bitmap
  one         flat AND, one operand with a bitmap
  none        flat AND, no bitmap
  cand_bitmap candidate-driven, every probed operand with a dense bitmap
  cand_probe  candidate-driven, every probed operand with a bitmap of either tier, at least one of them a probe bitmap
  cand_dir    candidate-driven, at least one operand probed through its block directory with both tiers on
and times each class as its own device-resident batch (exec_batch_device, as bench.py; CUDA events over --steps steps after --warmup).
Per class it prints ms per step, (query, tile) work items (candidate-driven: lead-term groups), matches, result words, and a model of
the HBM traffic of bitmap reads:
  * flat ANDs: per-tile order (every item reads its operands' tile words) and run-major order (every bitmap run read once);
  * candidate-driven: the probes issued (an upper bound: every lead document against every other operand) and the 32-byte bitmap
    sectors they read — in query order (the 16 bitmaps are several times L2, so each query's probes read their own sectors: the
    expected distinct sectors of its lead documents in each bitmap) and in run-major order (the queries in flight share a docID window,
    so each bitmap sector is read once per batch: the expected distinct sectors of all the class's probes of that bitmap).
Probes of the probe tier and of the directory are counted, not modelled.  Needs a GPU; prints the card and its power limit.

    python scripts/and2_breakdown.py [--ndocs 100000000] [--steps 20] [--warmup 5] [--settings runs,probe_off,cand_query_order]
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


SETTINGS = {"runs": {}, "probe_off": {"TRN_PROBE_BITMAPS": "0"}, "cand_query_order": {"TRN_CAND_RUNS": "0"}, "mixed_tiles": {"TRN_MIXED_RUNS": "0"},
            "tiles": {"TRN_DENSE_RUNS": "0", "TRN_MIXED_RUNS": "0"}}


def distinct_sectors(probes, sectors):
    """expected distinct sectors hit by `probes` uniformly spread probes over `sectors` sectors"""
    return sectors * -np.expm1(-probes / sectors) if sectors else 0.0


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
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the sources per class")
    ap.add_argument("--settings", default="runs,probe_off,cand_query_order", help=f"comma-separated sources to time, of {list(SETTINGS)}")
    args = ap.parse_args()
    settings = {k: SETTINGS[k] for k in args.settings.split(",")}
    import torch

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    synth = tb.SynthIndex(tb.CODEC_GOOGLE, args.ndocs, args.nterms, threads=max(1, len(os.sched_getaffinity(0))))
    srcs = {k: source(synth, args.ndocs, env) for k, env in settings.items()}
    g = next(iter(srcs.values()))
    texts, _ = bench.gen_queries("and2", args.nq, args.nterms)
    tdict = tb.TermDictionary(synth.names)
    plans = [tb.parse_query(q, tdict) for q in texts]
    terms = np.asarray(synth.terms)
    # the probe tier of the default settings, selected on the host as the upload does (the probed offset of a dense term is its dense one)
    env = {k: os.environ.pop(k) for k in ("TRN_PROBE_BITMAPS", "TRN_PROBE_RATIO", "TRN_PROBE_BUDGET", "TRN_DENSE_BITMAPS", "TRN_DENSE_BUDGET") if k in os.environ}
    probe_off, _, _ = tb.debug_probe_terms(tb.CODEC_GOOGLE, np.asarray(synth.index), terms)
    os.environ.update(env)
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
    classes = {"both": [], "one": [], "none": [], "cand_bitmap": [], "cand_probe": [], "cand_dir": []}
    in_probe_tier = lambda t: probe_off[t] != tb.DENSE_NONE and not bitmap_bytes(t)
    docs = lambda t: int(terms["documents"][t])
    for i, p in enumerate(plans):
        ts = [int(x["term"]) for x in p if x["kind"] == tb.NODE_TERM]
        nd = sum(bitmap_bytes(t) > 0 for t in ts)
        if routes[i] == tb.ROUTE_CANDIDATE:
            # a model of the planner's choice, not the planner's own: the rarest term (by blocks) leads (and2: both terms are necessary);
            # plan_batch breaks a tie in block counts by an unstable sort, so on a tie its lead may be the other term
            lead = min(ts, key=lambda t: (-(-docs(t) // 32), ts.index(t)))
            probed = [t for t in ts if t != lead]
            cls = "cand_bitmap" if all(bitmap_bytes(t) for t in probed) else "cand_probe" if all(bitmap_bytes(t) or in_probe_tier(t) for t in probed) else "cand_dir"
            classes[cls].append(i)
        elif routes[i] == tb.ROUTE_FLAT_AND:
            classes["both" if nd == len(ts) else "one" if nd else "none"].append(i)
    print(json.dumps({"card": card, "ndocs": args.ndocs, "nq": args.nq, "dense_terms": g.info()["dense_terms"],
                      "dense_bitmap_bytes": g.info()["dense_bitmap_bytes"],
                      **{f"probe_{f}_{k}": s.info()[f"probe_{f}"] for k, s in srcs.items() for f in ("terms", "bitmap_bytes")}}))
    stream = torch.cuda.current_stream()
    for name, qs in classes.items():
        if not qs:
            continue
        sub = [plans[i] for i in qs]
        items = old_b = 0
        used = set()
        probes = dir_probes = tier_probes = 0
        sec_query = 0.0
        per_bitmap = {}  # bitmap term -> probes of the class against it
        for i in qs:
            ts = [int(x["term"]) for x in plans[i] if x["kind"] == tb.NODE_TERM]
            if name.startswith("cand"):  # 32-block groups of the lead (rarest) term
                lead = min(ts, key=lambda t: (-(-docs(t) // 32), ts.index(t)))  # (the model of the lead above)
                lead_blocks = -(-docs(lead) // 32)
                items += -(-lead_blocks // 32)
                for t in ts:
                    if t == lead:
                        continue
                    probes += docs(lead)
                    if bitmap_bytes(t):
                        sec_query += distinct_sectors(docs(lead), bitmap_bytes(t) // 32)
                        per_bitmap[t] = per_bitmap.get(t, 0) + docs(lead)
                    elif in_probe_tier(t):
                        tier_probes += docs(lead)
                    else:
                        dir_probes += docs(lead)
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
        row = {"class": name, "queries": len(qs), "work_items": items, "matches": int(res.match_counts.sum()),
               "result_bytes": res.result_bytes(), **{f"ms_per_step_{k}": [round(x, 3) for x in v] for k, v in ms.items()},
               **{f"ms_median_{k}": round(float(np.median(v)), 3) for k, v in ms.items()}}
        if name.startswith("cand"):
            sec_run = sum(distinct_sectors(n, bitmap_bytes(t) // 32) for t, n in per_bitmap.items())
            row.update({"probes_upper_bound": probes, "probe_tier_probes_upper_bound": tier_probes, "directory_probes_upper_bound": dir_probes, "bitmap_sectors_query_order": round(sec_query),
                        "bitmap_sectors_run_major": round(sec_run), "bitmap_bytes_query_order": round(sec_query) * 32,
                        "bitmap_bytes_run_major": round(sec_run) * 32})
        else:
            row.update({"bitmap_bytes_per_tile_order": old_b, "bitmap_bytes_run_major": new_b})
        print(json.dumps(row))
    for s in srcs.values():
        s.close()


if __name__ == "__main__":
    main()
