#!/usr/bin/env python
"""Where the warps of tcx_first_kernel spend their time (needs a GPU).

    python scripts/first_kernel_timeline.py [--lib PATH] [--out FILE.json]

Builds the AG_FIRST_TIMELINE variant with scripts/build_variant.sh (or loads --lib), runs the default bench.py pipeline (16 x 1024x768,
K = 2000, AffNet + OriNet + HardNet) once to warm up and once recorded, and prints, for each of the three tcx_first_kernel launches and
each warpgroup, the share of the kernel's SM cycles its warps spent in each state.  In the variant every warp of CTAs 0-3 adds up
clock64 cycles per state; the shares are over the warps' whole run in the kernel.  Consumers: waiting for the producers' P plane
(p_full), issuing MMAs, wgmma_wait (their own MMAs), the warpgroup barrier (layer 2's row exchange), the barriers of both warpgroups
between layers, and the rest (epilogues, loop control).  Producers: waiting for the consumers to free a P half (p_empty), barrier 1
(input_norm's reductions), building the P planes, and the rest (sampling, input_norm).
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

STATES = ["total", "wait_p", "issue", "mma_wait", "wg_bar", "stage_bar", "p_build"]   # TL_* in tcx_first.cuh
CONSUMER = [("wait for P (p_full)", "wait_p"), ("issue MMAs", "issue"), ("wait for own MMAs", "mma_wait"),
            ("warpgroup barrier", "wg_bar"), ("both-warpgroup barriers", "stage_bar")]
PRODUCER = [("wait for a free P half (p_empty)", "wait_p"), ("barrier 1 (input_norm)", "wg_bar"), ("build P planes", "p_build")]
LAUNCHES = ["AffNet", "OriNet", "HardNet"]   # launch order of one pipeline step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="an AG_FIRST_TIMELINE build (default: build one with scripts/build_variant.sh)")
    ap.add_argument("--out", default=None, help="also write the shares as JSON")
    args = ap.parse_args()
    lib_path = args.lib
    if lib_path is None:
        subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_variant.sh"), "timeline", "-DAG_FIRST_TIMELINE"], check=True)
        lib_path = os.path.join(ROOT, "affnet_b200", "lib", "libaffnet_b200_timeline.so")
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

    read = L.lib().ag_first_timeline_read
    read.restype, read.argtypes = C.c_int, [C.c_void_p, C.c_void_p, C.c_int]
    dims = np.zeros(3, np.int32)
    assert read(None, dims.ctypes.data, 1) == 0
    n_launch, n_cta, n_state = (int(v) for v in dims)
    pipe.run(imgs)                       # warm-up (module load, first launches)
    torch.cuda.synchronize()
    assert read(None, None, 1) == 0
    pipe.run(imgs)
    torch.cuda.synchronize()
    buf = np.zeros((n_launch, n_cta, 16, n_state), np.uint64)
    assert read(buf.ctypes.data, None, 1) == 0
    buf = buf.astype(np.float64)
    ix = {s: i for i, s in enumerate(STATES)}

    props = torch.cuda.get_device_properties(0)
    report = {"gpu": props.name, "ctas_recorded": n_cta, "kernels": {}}
    print("%s: shares of each warp's cycles in tcx_first_kernel, CTAs 0-%d, default bench.py pipeline" % (props.name, n_cta - 1))
    for li, name in enumerate(LAUNCHES):
        kern = {"cycles_per_cta": float(buf[li, :, :, ix["total"]].max(axis=1).mean())}
        for role, warps, rows in (("producers (warps 0-7)", range(0, 8), PRODUCER),
                                  ("consumer warpgroup 0 (warps 8-11)", range(8, 12), CONSUMER),
                                  ("consumer warpgroup 1 (warps 12-15)", range(12, 16), CONSUMER)):
            sel = buf[li][:, list(warps), :].sum(axis=(0, 1))
            tot = sel[ix["total"]]
            shares = {label: sel[ix[key]] / tot for label, key in rows}
            shares["rest (epilogues / sampling, loop control)"] = 1.0 - sum(shares.values())
            kern[role] = {k: round(float(v), 4) for k, v in shares.items()}
        report["kernels"][name] = kern
        print("\n%s  (%.0f cycles per CTA)" % (name, kern["cycles_per_cta"]))
        for role in [k for k in kern if k != "cycles_per_cta"]:
            print("  " + role)
            for k, v in kern[role].items():
                print("    %-44s %5.1f %%" % (k, 100 * v))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
