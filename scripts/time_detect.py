"""Device time of the detector (ag_detect: detect_rows_kernel + resolve_kernel) on the bench workload (config 2: 16 images of 768x1024,
bench.py's images, nlevels 3, border 5), measured with CUDA events over many launches.

    python scripts/time_detect.py [--other TREE] [--rounds R] [--iters N]

With --other, the same measurement of TREE's library (another checkout of this repository, built) alternates with this tree's, one
process per measurement, so that two builds are compared under the same conditions.  Prints one line per measurement and the
median of each build, with the GPU's name and power limit."""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def measure(iters):
    import ctypes as C
    import torch
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import affnet_b200._lib as L
    from bench import make_images
    from helpers import Detector, gpu_pyramids
    imgs = make_images(16, 1234, 768, 1024)
    plan, buf, _ = gpu_pyramids(L, imgs, 3, 5)
    det = Detector(L, plan, buf)
    lib = L.lib()
    call = lambda: L.check(lib.ag_detect(C.byref(plan), L.ptr(buf), 0.0, 5, C.byref(det.ws), L.stream_ptr()))  # noqa: E731
    for _ in range(20):
        call()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        call()
    t1.record()
    torch.cuda.synchronize()
    print("%.4f" % (t0.elapsed_time(t1) / iters))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", default=None)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        measure(a.iters)
        return
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    builds = {"this": os.path.join(ROOT, "affnet_b200", "lib", "libaffnet_b200.so")}
    if a.other:
        builds["other"] = os.path.join(os.path.abspath(a.other), "affnet_b200", "lib", "libaffnet_b200.so")
    times = {k: [] for k in builds}
    for r in range(a.rounds):
        for k in (list(builds) if r % 2 == 0 else list(builds)[::-1]):
            env = dict(os.environ, AFFNET_B200_LIB=builds[k])
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--iters", str(a.iters)], env=env, capture_output=True,
                                 text=True, check=True).stdout.split()[-1]
            times[k].append(float(out))
            print("round %d %-5s %s ms" % (r, k, out), flush=True)
    for k, v in times.items():
        print("%s: median %.4f ms, min %.4f, max %.4f per ag_detect call (16 x 768x1024), %s" % (k, statistics.median(v), min(v), max(v), gpu))


if __name__ == "__main__":
    main()
