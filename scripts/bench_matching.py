"""Batched SNN matching (Losses.match_snn_pairs, ag_match_pairs) against today's practice (a Python loop of Losses.match_snn over
count-sliced descriptors, the counts read to the host first) on the pipeline's own outputs.  Workloads: 16 x 1024x768 synthetic images at
K = 2000 (the 15 consecutive pairs and the 240 ordered pairs i != j) and 64 x 1920x1080 at K = 4000 (the 63 consecutive pairs).
Batched: CUDA-event time of a CUDA-graph replay of the one call (median of --steps after --warmup).  Loop: host clock from before the
count read to a device synchronise (median of --steps after --warmup).  The two must agree bit for bit (tentatives, min and second
distances).  Achieved FLOP/s counts 2 passes x 2 n1 n2 D over the actual counts, against the data sheet's 67 TFLOP/s FP32 of the H100
SXM.  The card's name and power limit are read in the same run.

    python scripts/bench_matching.py [--steps 20] [--warmup 5] [--out FILE.json]

Needs an H100 (there is no CPU path); prints one JSON document.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

FP32_PEAK = 67e12   # H100 SXM data sheet, dense FP32 (700 W card)
WORKLOADS = [
    # name, B, H, W, K, {pair set: [(i, j), ...]}
    ("16 x 1024x768, K = 2000", 16, 768, 1024, 2000, {"15 consecutive pairs": [(i, i + 1) for i in range(15)],
                                                       "240 ordered pairs": [(i, j) for i in range(16) for j in range(16) if i != j]}),
    ("64 x 1920x1080, K = 4000", 64, 1080, 1920, 4000, {"63 consecutive pairs": [(i, i + 1) for i in range(63)]}),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(name=torch.cuda.get_device_name(), nvidia_smi=q)


def describe(nets, B, H, Wd, K, chunk=16):
    """Descriptors [B,K,128] and counts [B] of B synthetic images, computed by the pipeline in batches of `chunk`."""
    from affnet_b200.pipeline import DetectDescribePipeline
    from helpers import synthetic_image
    a, o, h = nets
    desc = torch.empty(B, K, 128, device="cuda")
    cnt = torch.empty(B, dtype=torch.int32, device="cuda")
    lafs = torch.empty(B, K, 2, 3, device="cuda")
    for b0 in range(0, B, chunk):
        n = min(chunk, B - b0)
        pipe = DetectDescribePipeline(n, H, Wd, a, h, o, num_features=K, outputs=[(lafs[b0:b0 + n], desc[b0:b0 + n], cnt[b0:b0 + n])])
        pipe.run(torch.cat([synthetic_image(H, Wd, 1234 + b0 + i) for i in range(n)]).cuda())
        pipe.check()
        del pipe
    torch.cuda.synchronize()
    return desc, cnt


def loop_match(desc, cnt, pairs, ratio):
    """Today's practice: the counts to the host, then one match_snn per pair on the count-sliced descriptors."""
    from affnet_b200.Losses import match_snn
    c = cnt.tolist()
    return [match_snn(desc[i, :c[i]], desc[j, :c[j]], ratio) for i, j in pairs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_matching.py needs a CUDA device")
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.Losses import match_snn_pairs
    from helpers import load_weights
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    nets = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    ratio = 0.8
    res = dict(card=card(), steps=args.steps, warmup=args.warmup, fp32_peak_tflops=FP32_PEAK / 1e12, workloads={})
    for wname, B, H, Wd, K, pairsets in WORKLOADS:
        desc, cnt = describe(nets, B, H, Wd, K)
        c = cnt.tolist()
        wres = res["workloads"][wname] = dict(keypoints_per_image_min=min(c), keypoints_per_image_max=max(c), pair_sets={})
        for pname, pl in pairsets.items():
            pairs = torch.tensor(pl, dtype=torch.int32, device="cuda")
            flops = sum(2 * 2 * c[i] * c[j] * 128 for i, j in pl)
            # batched: one call, captured in a CUDA graph
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                match_snn_pairs(desc, cnt, pairs=pairs, SNN_threshold=ratio)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = match_snn_pairs(desc, cnt, pairs=pairs, SNN_threshold=ratio)
            for _ in range(args.warmup):
                g.replay()
            torch.cuda.synchronize()
            bms = []
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                e1.synchronize()
                bms.append(e0.elapsed_time(e1))
            bms.sort()
            # today's practice
            for _ in range(args.warmup):
                loop_match(desc, cnt, pl, ratio)
            torch.cuda.synchronize()
            lms = []
            for _ in range(args.steps):
                t0 = time.perf_counter()
                ref = loop_match(desc, cnt, pl, ratio)
                torch.cuda.synchronize()
                lms.append((time.perf_counter() - t0) * 1e3)
            lms.sort()
            tent, ntent, mn, sec = out
            nt = ntent.tolist()
            for p, ((i, j), (i1, i2, omn, osec)) in enumerate(zip(pl, ref)):
                assert nt[p] == i1.numel(), (wname, pname, p, nt[p], i1.numel())
                assert torch.equal(tent[p, :nt[p], 0].long(), i1) and torch.equal(tent[p, :nt[p], 1].long(), i2), (wname, pname, p)
                assert torch.equal(mn[p, :c[i]], omn) and torch.equal(sec[p, :c[i]], osec), (wname, pname, p)
            b, lp = bms[len(bms) // 2], lms[len(lms) // 2]
            wres["pair_sets"][pname] = dict(
                pairs=len(pl), tentatives=sum(nt), bit_identical_to_loop=True, flop=flops,
                batched_graph_ms_median=b, batched_graph_ms_min=bms[0], batched_graph_ms_max=bms[-1],
                batched_tflops=flops / (b * 1e-3) / 1e12, batched_share_of_fp32_peak=flops / (b * 1e-3) / FP32_PEAK,
                loop_ms_median=lp, loop_ms_min=lms[0], loop_ms_max=lms[-1], loop_tflops=flops / (lp * 1e-3) / 1e12,
                speedup_loop_over_batched=lp / b)
            print("%-26s %-22s batched %8.3f ms (%5.1f TFLOP/s)   loop %8.3f ms   x%.2f" % (
                wname, pname, b, flops / (b * 1e-3) / 1e12, lp, lp / b), file=sys.stderr)
            del g, out, ref
        del desc, cnt
        torch.cuda.empty_cache()
    res["card"]["after"] = card()["nvidia_smi"]
    doc = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
