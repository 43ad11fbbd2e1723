#!/usr/bin/env python
"""Where the warps of tcx_conv_kernel spend their time (needs a GPU).

    python scripts/conv_kernel_timeline.py [--lib PATH] [--out FILE.json] [--old-schedule]

Builds the AG_CONV_TIMELINE variant with scripts/build_variant.sh (--old-schedule: with AG_CONV_PINGPONG=0 as well), or loads --lib,
runs the default bench.py pipeline (16 x 1024x768, K = 2000, AffNet + OriNet + HardNet) once to warm up and once recorded, and prints,
for each of the ten tcx_conv_kernel launches of a step (labelled by net and layer), the share of the kernel's SM cycles the warps of
each role spent in each state.  In the variant every warp of the split-0 CTAs 0-3 adds up clock64 cycles per state.  Consumers:
waiting for the loader (full), waiting for their turn to issue (ping-pong only), issuing MMAs, wgmma_wait on their own MMAs, the
epilogue, the warpgroup barrier before a stage is released (previous schedule only), and the rest (loop control).  Loader: waiting
for a free stage (empty), and the rest (issuing the bulk copies).

Warp 0 of each consumer warpgroup of CTA 0 also logs, per block, when its MMA issue starts, when its MMAs have completed and when
its epilogue ends.  From those the script reports, per launch: the share of each warpgroup's epilogue time during which the other
warpgroup was in an epilogue too, and the share of CTA 0's run during which neither warpgroup had MMAs issued and not yet waited for
(an upper bound on the tensor core's idle time).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

STATES = ["total", "wait_full", "turn", "issue", "mma_wait", "epilogue", "wg_bar", "wait_empty", "other"]   # CT_* in tcx_conv.cuh
CONSUMER = [("wait for the loader (full)", "wait_full"), ("wait for the turn (ping-pong)", "turn"), ("issue MMAs", "issue"),
            ("wait for own MMAs", "mma_wait"), ("epilogue", "epilogue"), ("warpgroup barrier", "wg_bar")]
LOADER = [("wait for a free stage (empty)", "wait_empty")]
LAUNCHES = ["AffNet L4", "AffNet L5", "AffNet L6", "OriNet L4", "OriNet L5", "OriNet L6",
            "HardNet L3", "HardNet L4", "HardNet L5", "HardNet L6"]   # launch order of one pipeline step


def overlap(a, b):
    """Total length of the intersection of two lists of disjoint intervals (arrays [n, 2])."""
    import numpy as np
    if len(a) == 0 or len(b) == 0:
        return 0.0
    lo = np.maximum(a[:, None, 0], b[None, :, 0])
    hi = np.minimum(a[:, None, 1], b[None, :, 1])
    return float(np.clip(hi - lo, 0, None).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="an AG_CONV_TIMELINE build (default: build one with scripts/build_variant.sh)")
    ap.add_argument("--old-schedule", action="store_true", help="build the variant with the previous schedule (AG_CONV_PINGPONG=0)")
    ap.add_argument("--out", default=None, help="also write the shares as JSON")
    args = ap.parse_args()
    lib_path = args.lib
    if lib_path is None:
        name, flags = ("conv_timeline_old", "-DAG_CONV_TIMELINE -DAG_CONV_PINGPONG=0") if args.old_schedule else ("conv_timeline", "-DAG_CONV_TIMELINE")
        subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_variant.sh"), name, flags], check=True)
        lib_path = os.path.join(ROOT, "affnet_b200", "lib", "libaffnet_b200_%s.so" % name)
    os.environ["AFFNET_B200_LIB"] = os.path.abspath(lib_path)

    import numpy as np
    import torch
    from helpers import load_weights, synthetic_image
    import affnet_b200._lib as L
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline

    H, W, K, border, B = 768, 1024, 2000, 5, 16   # bench.py --config 2
    w = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(w["affnet"]); o.load_state_dict(w["orinet"]); h.load_state_dict(w["hardnet"])
    a, o, h = a.eval().cuda(), o.eval().cuda(), h.eval().cuda()
    imgs = torch.cat([synthetic_image(H, W, 1234 + i) for i in range(B)]).cuda()
    pipe = DetectDescribePipeline(B, H, W, a, h, o, num_features=K, border=border, do_ori=True)

    read = L.lib().ag_conv_timeline_read
    read.restype, read.argtypes = C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    dims = np.zeros(4, np.int32)
    assert read(None, None, dims.ctypes.data, 1) == 0
    n_launch, n_cta, n_state, n_ev = (int(v) for v in dims)
    pipe.run(imgs)                       # warm-up (module load, first launches)
    torch.cuda.synchronize()
    assert read(None, None, None, 1) == 0
    pipe.run(imgs)
    torch.cuda.synchronize()
    sums = np.zeros((n_launch, n_cta, 9, n_state), np.uint64)
    ev = np.zeros((n_launch, 2, n_ev, 3), np.uint64)
    assert read(sums.ctypes.data, ev.ctypes.data, None, 1) == 0
    sums = sums.astype(np.float64)
    ix = {s: i for i, s in enumerate(STATES)}

    props = torch.cuda.get_device_properties(0)
    report = {"gpu": props.name, "ctas_recorded": n_cta, "kernels": {}}
    print("%s: shares of each warp's cycles in tcx_conv_kernel, split-0 CTAs 0-%d, default bench.py pipeline" % (props.name, n_cta - 1))
    for li, name in enumerate(LAUNCHES):
        kern = {"cycles_per_cta": float(sums[li, :, :, ix["total"]].max(axis=1).mean())}
        for role, warps, rows in (("consumer warpgroup 0 (warps 0-3)", range(0, 4), CONSUMER),
                                  ("consumer warpgroup 1 (warps 4-7)", range(4, 8), CONSUMER),
                                  ("loader (warp 8)", [8], LOADER)):
            sel = sums[li][:, list(warps), :].sum(axis=(0, 1))
            tot = sel[ix["total"]]
            shares = {label: sel[ix[key]] / tot for label, key in rows}
            shares["rest (loop control%s)" % ("" if role.startswith("consumer") else ", bulk copies")] = 1.0 - sum(shares.values())
            kern[role] = {k: round(float(v), 4) for k, v in shares.items()}
        # CTA 0's block events: [issue start, MMAs done, epilogue end] per block and warpgroup
        blk = [e[e[:, 2] > 0].astype(np.float64) for e in ev[li]]
        if all(len(b) for b in blk):
            t0 = min(b[:, 0].min() for b in blk)
            t1 = max(b[:, 2].max() for b in blk)
            epi = [b[:, 1:3] for b in blk]
            mma = [b[:, 0:2] for b in blk]
            both = overlap(epi[0], epi[1])
            busy = sum(float((m[:, 1] - m[:, 0]).sum()) for m in mma) - overlap(mma[0], mma[1])
            kern["CTA 0"] = {
                "blocks per warpgroup": [len(b) for b in blk],
                "epilogue share of the run, per warpgroup": [round(float((e[:, 1] - e[:, 0]).sum()) / (t1 - t0), 4) for e in epi],
                "share of each warpgroup's epilogue time with the other in an epilogue too": [round(both / float((e[:, 1] - e[:, 0]).sum()), 4) for e in epi],
                "share of the run with no MMAs in flight": round(1.0 - busy / (t1 - t0), 4),
            }
        report["kernels"][name] = kern
        print("\n%s  (%.0f cycles per CTA)" % (name, kern["cycles_per_cta"]))
        for role in [k for k in kern if k not in ("cycles_per_cta", "CTA 0")]:
            print("  " + role)
            for k, v in kern[role].items():
                print("    %-44s %5.1f %%" % (k, 100 * v))
        if "CTA 0" in kern:
            print("  CTA 0, warp 0 of each warpgroup")
            for k, v in kern["CTA 0"].items():
                if k == "blocks per warpgroup":
                    print("    %-72s %s" % (k, v))
                elif isinstance(v, list):
                    print("    %-72s %s" % (k, " / ".join("%5.1f %%" % (100 * x) for x in v)))
                else:
                    print("    %-72s %5.1f %%" % (k, 100 * v))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
