"""Developer tool: digest of an `ncu --page source --csv` export: executed warp instructions by opcode and the
hottest address ranges (executed count x stall samples), to see where a SIMT kernel's issue slots go.
    python scripts/src_hot.py <source-view export>.csv [top]"""
import csv
import sys
from collections import Counter


def main():
    path = sys.argv[1]
    top = int(sys.argv[2]) if len(sys.argv) > 2 else 25
    rows = list(csv.reader(open(path)))
    hdr_i = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
    hdr = rows[hdr_i]
    col = {n: i for i, n in enumerate(hdr)}
    print(rows[0][:2])
    ops, samples = Counter(), Counter()
    tot = tot_s = 0
    recs = []
    for r in rows[hdr_i + 1:]:
        if len(r) < len(hdr) or not r[col["Instructions Executed"]].strip():
            continue
        n = int(r[col["Instructions Executed"]])
        s = int(r[col["# Samples"]] or 0)
        src = r[col["Source"]].strip()
        op = src.split()[0] if not src.startswith("@") else src.split()[1]
        op = op.split(".")[0].rstrip(";")
        ops[op] += n
        samples[op] += s
        tot += n
        tot_s += s
        recs.append((r[col["Address"]], n, s, src, float(r[col["Avg. Threads Executed"]] or 0)))
    print("executed warp instructions: %d, samples %d" % (tot, tot_s))
    for op, n in ops.most_common(top):
        print("  %-12s %6.2f %% of instructions  %6.2f %% of samples" % (op, 100.0 * n / tot, 100.0 * samples[op] / max(tot_s, 1)))
    # contiguous regions by executed count (basic blocks): group consecutive instructions with equal executed count
    blocks = []
    cur = None
    for a, n, s, src, thr in recs:
        if cur and cur["n"] == n:
            cur["k"] += 1; cur["s"] += s; cur["thr"] += thr
        else:
            cur = {"a": a, "n": n, "k": 1, "s": s, "first": src, "thr": thr}
            blocks.append(cur)
    blocks.sort(key=lambda b: -b["n"] * b["k"])
    print("hottest blocks (instructions x executions):")
    for b in blocks[:top]:
        print("  %s  %4d instr x %9d exec = %5.2f %% of issue, %5.2f %% of samples, avg threads %.1f | %s" % (
            b["a"], b["k"], b["n"], 100.0 * b["n"] * b["k"] / tot, 100.0 * b["s"] / max(tot_s, 1), b["thr"] / b["k"], b["first"][:60]))


if __name__ == "__main__":
    main()
