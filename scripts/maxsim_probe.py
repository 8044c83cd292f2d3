"""Where the headline max-sim kernel's time goes: the bench's ColBERT inputs (same seed, shapes and on-GPU generation as
`bench.py --workload colbert`) timed under these variants, alternated in rounds, with CUDA events per launch.

    masked       maxsim(..., impl="tcgen05") with both masks, exactly as bench.py runs it
    nomask       the same tensors with q_mask = d_mask = None: every row of every document is live (scores differ)
    ragged       impl="tcgen05_ragged" (the live-row fetch by its historical name)
    ragged_full  impl="tcgen05_ragged" with an all-ones document mask, next to
    dense_full   impl="tcgen05" on that same mask: equal bytes, so the difference is the cost of the ragged bookkeeping
    compact      impl="tcgen05" on a copy of the documents re-laid out at Ld = --compact-ld (about the mean fetched rows),
                 masks cut to match: the same kernel over about the live bytes.  Scores differ; it is a ceiling for timing
    compact_nomask  that copy with q_mask = d_mask = None: the same bytes with no mask loads, so the difference to
                 `compact` is what the mask path costs
    train        impl="tcgen05" with return_argmax=True, the training instantiation
    read         a plain full read of the 2.95 GB document tensor (an fp32-accumulated sum): a rough attainable-bandwidth
                 reference, not the kernel's roof

    python scripts/maxsim_probe.py [--rounds 5] [--steps 20] [--out FILE] [--profile DIR]

Prints one JSON line per variant and a markdown table; --out also writes the JSON.  The SM clock is sampled through NVML
read-only queries while the timed rounds run, as in bench.py.  `live_gb_per_s` counts the document bytes a live-row fetch
reads (each document up to its last unmasked row, rounded up to 16 rows); `fetched_gb_per_s` the bytes the kernel
actually fetches: each document's rows [0, live), its end-aligned 64-row chunks zero-filling the rows below 0 without
reading HBM.  Against the debugging build (`python -m matchmaker_b200.build --prof`) with
MMB200_MAXSIM_PROF=1, the library prints the kernel's per-role cycle counters after every launch (`--rounds 1 --steps 1`
keeps that to four launches per variant).  --profile runs a separate torch.profiler pass
afterwards (a few launches of each max-sim variant) and prints every kernel each variant launches with its device time
and the gap between consecutive kernels of one call.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from matchmaker_b200 import interaction  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="launches per variant per round")
    ap.add_argument("--ld", type=int, default=None,
                    help="document length other than the bench's 180 (e.g. 220: the 256-row tile of the kernel)")
    ap.add_argument("--compact-ld", type=int, default=83, help="padded length of the `compact` variant's copy")
    ap.add_argument("--variants", default=None, help="comma-separated subset of the variants")
    ap.add_argument("--profile", default=None, metavar="DIR", help="also run a torch.profiler pass, trace under DIR")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.ld is not None:   # same generator, other padded length; the algorithmic bytes follow it
        bench.LD = args.ld

    assert torch.cuda.is_available(), "the probe times GPU kernels; there is no CPU path"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    wl = bench.ColbertWorkload(0, dev)
    wl.to_device()
    dpq = bench.DOCS_PER_QUERY
    wl.alg_bytes = (bench.LD * bench.DIM * 2 + 4 + 4 + (bench.LQ * bench.DIM * 2) // dpq) * wl.pairs
    full_dm = torch.ones_like(wl.cdm)
    cl = min(args.compact_ld, bench.LD)
    compact_d, compact_dm = wl.cd[:, :cl].contiguous(), wl.cdm[:, :cl].contiguous()
    # document bytes of the live-row fetch: rows up to the last unmasked one, in 16-row blocks
    idx = torch.arange(1, bench.LD + 1, device=dev)
    live = (wl.cdm.to(torch.int64) * idx).amax(dim=1)
    live_bytes = int(((live + 15) // 16 * 16).clamp(max=bench.LD).sum().item()) * bench.DIM * 2

    def fetched_bytes(dm, ld):
        """Document bytes the kernel fetches: rows [0, live) of each document (its end-aligned chunks zero-fill the rows
        below 0 without reading HBM); live = ld without a mask."""
        if dm is None:
            return wl.cd.shape[0] * ld * bench.DIM * 2
        lv = (dm.to(torch.int64) * torch.arange(1, ld + 1, device=dev)).amax(dim=1)
        return int(lv.sum().item()) * bench.DIM * 2

    variants = {
        "masked": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, wl.cdm, docs_per_query=dpq, impl="tcgen05"),
        "nomask": lambda: interaction.maxsim(wl.cq, wl.cd, None, None, docs_per_query=dpq, impl="tcgen05"),
        "ragged": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, wl.cdm, docs_per_query=dpq, impl="tcgen05_ragged"),
        "ragged_full": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, full_dm, docs_per_query=dpq, impl="tcgen05_ragged"),
        "dense_full": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, full_dm, docs_per_query=dpq, impl="tcgen05"),
        "compact": lambda: interaction.maxsim(wl.cq, compact_d, wl.cqm, compact_dm, docs_per_query=dpq, impl="tcgen05"),
        "compact_nomask": lambda: interaction.maxsim(wl.cq, compact_d, None, None, docs_per_query=dpq, impl="tcgen05"),
        "train": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, wl.cdm, docs_per_query=dpq, impl="tcgen05",
                                            return_argmax=True),
        "read": lambda: wl.cd.sum(dtype=torch.float32),
    }
    if args.variants:
        variants = {k: variants[k] for k in args.variants.split(",")}
    # document bytes each variant reads from HBM
    var_bytes = {"masked": wl.cd.numel() * 2, "nomask": wl.cd.numel() * 2, "ragged": live_bytes,
                 "ragged_full": wl.cd.numel() * 2, "dense_full": wl.cd.numel() * 2, "compact": compact_d.numel() * 2,
                 "compact_nomask": compact_d.numel() * 2, "train": wl.cd.numel() * 2, "read": wl.cd.numel() * 2}
    # document bytes each max-sim variant actually fetches (the live-row chunks of its masks)
    var_fetched = {"masked": fetched_bytes(wl.cdm, bench.LD), "nomask": fetched_bytes(None, bench.LD),
                   "ragged": fetched_bytes(wl.cdm, bench.LD), "ragged_full": fetched_bytes(full_dm, bench.LD),
                   "dense_full": fetched_bytes(full_dm, bench.LD), "compact": fetched_bytes(compact_dm, cl),
                   "compact_nomask": fetched_bytes(None, cl), "train": fetched_bytes(wl.cdm, bench.LD)}
    for name, f in variants.items():
        if os.environ.get("MMB200_MAXSIM_PROF"):   # a debugging build prints its counters after each launch
            print("maxsim_prof variant %s" % name, file=sys.stderr, flush=True)
        for _ in range(3):
            f()
    torch.cuda.synchronize()

    samples = {k: [] for k in variants}
    sampler = bench.ClockSampler(0)
    sampler.start()
    t0 = time.perf_counter()
    for r in range(args.rounds):
        names = list(variants) if r % 2 == 0 else list(reversed(variants))
        for name in names:
            f = variants[name]
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for a, b in ev:
                a.record()
                f()
                b.record()
            torch.cuda.synchronize()
            samples[name] += [a.elapsed_time(b) for a, b in ev]
    clocks = sampler.stop([(t0, time.perf_counter())])

    doc_bytes = wl.cd.numel() * wl.cd.element_size()
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "clocks": clocks, "Ld": bench.LD,
           "rounds": args.rounds, "steps_per_round": args.steps, "pairs": wl.pairs, "alg_bytes": wl.alg_bytes,
           "doc_bytes": doc_bytes, "live_bytes": live_bytes, "compact_ld": cl, "variants": {}}
    for name, ts in samples.items():
        med = statistics.median(ts)
        rec = {"median_ms": med, "min_ms": min(ts), "max_ms": max(ts), "n": len(ts)}
        if name == "read":
            rec["gb_per_s"] = doc_bytes / (med * 1e-3) / 1e9
        else:
            rec["pairs_per_s"] = wl.pairs / (med * 1e-3)
            rec["alg_gb_per_s"] = wl.alg_bytes / (med * 1e-3) / 1e9
            rec["us_per_doc_per_sm"] = med * 1e3 / (wl.pairs / torch.cuda.get_device_properties(dev).multi_processor_count)
            rec["doc_gb_per_s"] = var_bytes[name] / (med * 1e-3) / 1e9
            rec["fetched_gb"] = var_fetched[name] / 1e9
            rec["fetched_gb_per_s"] = var_fetched[name] / (med * 1e-3) / 1e9
            if name in ("masked", "ragged", "train"):   # bytes a live-row fetch needs, over this variant's time
                rec["live_gb_per_s"] = live_bytes / (med * 1e-3) / 1e9
        res["variants"][name] = rec
        print(json.dumps({name: rec}), flush=True)

    print("card: %s, power limit %s W, SM clock median %s MHz (max %s), Ld %d" % (
        res["card"], res["power_limit_w"], clocks.get("sm_mhz"), clocks.get("sm_max_mhz"), bench.LD))
    print("live-row bytes %.3f GB of %.3f GB; compact copy %.3f GB (Ld %d)" % (
        live_bytes / 1e9, doc_bytes / 1e9, compact_d.numel() * 2 / 1e9, cl))
    print("| variant | median ms | min | max | pairs/s | GB/s (algorithmic; `read`: tensor bytes) | document GB/s read "
          "| GB fetched | fetched GB/s |")
    print("|---|---|---|---|---|---|---|---|---|")
    for name, rec in res["variants"].items():
        gbs = rec.get("alg_gb_per_s", rec.get("gb_per_s"))
        pps = "%.3g" % rec["pairs_per_s"] if "pairs_per_s" in rec else "-"
        dgb = rec.get("doc_gb_per_s", rec.get("gb_per_s"))
        fgb = "%.3f | %.0f" % (rec["fetched_gb"], rec["fetched_gb_per_s"]) if "fetched_gb" in rec else "- | -"
        print("| %s | %.3f | %.3f | %.3f | %s | %.0f | %.0f | %s |" % (name, rec["median_ms"], rec["min_ms"],
                                                                     rec["max_ms"], pps, gbs, dgb, fgb))
    if args.profile:
        res["profile"] = profile(variants, args.profile)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


def profile(variants, out_dir, calls=5):
    """Kernels of each max-sim variant under torch.profiler (a run of its own, after the timed rounds): per call, each
    kernel's device time and the idle gap before it on the device."""
    from torch.profiler import ProfilerActivity, profile as tprofile
    os.makedirs(out_dir, exist_ok=True)
    summary = {}
    for name, f in variants.items():
        if name == "read":
            continue
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            for _ in range(calls):
                f()
                torch.cuda.synchronize()
        prof.export_chrome_trace(os.path.join(out_dir, "probe_%s.pt.trace.json" % name))
        kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                      key=lambda e: e.time_range.start)
        per = {}
        prev_end = None
        for e in kern:
            gap = None if prev_end is None else e.time_range.start - prev_end
            prev_end = e.time_range.end
            r = per.setdefault(e.name, {"n": 0, "us": [], "gap_before_us": []})
            r["n"] += 1
            r["us"].append(e.time_range.end - e.time_range.start)
            if gap is not None and gap < 100:   # gaps inside one call (calls are separated by a synchronise)
                r["gap_before_us"].append(gap)
        summary[name] = {k: {"n": v["n"], "median_us": statistics.median(v["us"]),
                             "median_gap_before_us": statistics.median(v["gap_before_us"]) if v["gap_before_us"] else None}
                         for k, v in per.items()}
        print(json.dumps({"profile": name, "kernels": summary[name]}), flush=True)
    return summary


if __name__ == "__main__":
    main()
