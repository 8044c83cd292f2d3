"""Where the headline max-sim kernel's time goes: the bench's ColBERT inputs (same seed, shapes and on-GPU generation as
`bench.py --workload colbert`) timed under four variants, alternated in rounds, with CUDA events per launch.

    (a) masked   maxsim(..., impl="tcgen05") with both masks, exactly as bench.py runs it
    (b) nomask   the same tensors with q_mask = d_mask = None: no per-document metadata loads (scores differ)
    (c) ragged   impl="tcgen05_ragged": rows past each document's last unmasked row are not fetched
    (d) read     a plain full read of the 2.95 GB document tensor (an fp32-accumulated sum): a rough attainable-bandwidth
                 reference, not the kernel's roof

    python scripts/maxsim_probe.py [--rounds 5] [--steps 20] [--out FILE]

Prints one JSON line per variant and a markdown table; --out also writes the JSON.  The SM clock is sampled through NVML
read-only queries while the timed rounds run, as in bench.py.
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
    variants = {
        "masked": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, wl.cdm, docs_per_query=dpq, impl="tcgen05"),
        "nomask": lambda: interaction.maxsim(wl.cq, wl.cd, None, None, docs_per_query=dpq, impl="tcgen05"),
        "ragged": lambda: interaction.maxsim(wl.cq, wl.cd, wl.cqm, wl.cdm, docs_per_query=dpq, impl="tcgen05_ragged"),
        "read": lambda: wl.cd.sum(dtype=torch.float32),
    }
    for f in variants.values():
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
           "doc_bytes": doc_bytes, "variants": {}}
    for name, ts in samples.items():
        med = statistics.median(ts)
        rec = {"median_ms": med, "min_ms": min(ts), "max_ms": max(ts), "n": len(ts)}
        if name == "read":
            rec["gb_per_s"] = doc_bytes / (med * 1e-3) / 1e9
        else:
            rec["pairs_per_s"] = wl.pairs / (med * 1e-3)
            rec["alg_gb_per_s"] = wl.alg_bytes / (med * 1e-3) / 1e9
            rec["us_per_doc_per_sm"] = med * 1e3 / (wl.pairs / torch.cuda.get_device_properties(dev).multi_processor_count)
        res["variants"][name] = rec
        print(json.dumps({name: rec}), flush=True)

    print("card: %s, power limit %s W, SM clock median %s MHz (max %s), Ld %d" % (
        res["card"], res["power_limit_w"], clocks.get("sm_mhz"), clocks.get("sm_max_mhz"), bench.LD))
    print("| variant | median ms | min | max | pairs/s | GB/s (algorithmic; `read`: tensor bytes) |")
    print("|---|---|---|---|---|---|")
    for name, rec in res["variants"].items():
        gbs = rec.get("alg_gb_per_s", rec.get("gb_per_s"))
        pps = "%.3g" % rec["pairs_per_s"] if "pairs_per_s" in rec else "-"
        print("| %s | %.3f | %.3f | %.3f | %s | %.0f |" % (name, rec["median_ms"], rec["min_ms"], rec["max_ms"], pps, gbs))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
