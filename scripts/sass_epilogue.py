"""Developer tool: static SASS instructions of the tcx_first_kernel epilogues per output value, by instruction class.

    python scripts/sass_epilogue.py [affnet_b200/csrc/obj/nets_tcx.o]

Disassembles the object's sm_90a cubin with line information (cuobjdump -xelf, nvdisasm -gi) and assigns every instruction of each
tcx_first_kernel instantiation to the code it came from: the layer-1 / layer-2 epilogue lambdas of tcx_first.cuh, or layer 3's
xconv_block_epilogue (tcx_conv.cuh).  An instruction of a helper inlined into a helper (pack2 inside split_pack2, ...) carries only
its innermost call site, so it goes where that call site last went, else where the previous instruction went.  The MMA issue
instructions (HGMMA, WARPGROUP, R2UR) are left out.  The counts are static:
each unrolled copy of a body counts once, and a body's count is divided by the output values (fp32 results, each written as hi [+ lo])
that all its copies produce per thread."""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASSES = [
    ("FFMA/FADD/FMNMX", ("FFMA", "FADD", "FMUL", "FMNMX")),
    ("F2FP/HADD2.F32", ("F2FP", "HADD2", "HFMA2", "HMUL2", "PRMT")),
    ("SHFL", ("SHFL",)),
    ("FSEL/SEL", ("FSEL", "SEL")),
    ("STS/STSM/STG", ("STS", "STSM", "STG")),
    ("LDS/LDC", ("LDS", "LDC", "LDG")),
    ("BAR", ("BAR",)),
]
# name, template arguments <C1, COUT, SA, SW, OSA, BF, L3>
INSTS = [("AffNet / OriNet <16,16,1,1,1,0,1>", "16ELi16ELi1ELi1ELi1ELi0ELi1E"),
         ("(L3 = 0) <16,16,1,1,1,0,0>", "16ELi16ELi1ELi1ELi1ELi0ELi0E"),
         ("HardNet <32,32,0,1,0,0,0>", "32ELi32ELi0ELi1ELi0ELi0ELi0E"),
         ("HardNet bf16 <32,32,0,1,0,1,0>", "32ELi32ELi0ELi1ELi0ELi1ELi0E")]
# instructions of the MMA issue (descriptors to uniform registers, wgmma), which the scheduler interleaves with the epilogues
ISSUE = ("HGMMA", "WARPGROUP", "R2UR")
ANN = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
INS = re.compile(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_]*)(\.[A-Z0-9_.]+)?")


def body_lines(path):
    """(file base name, line) -> body, for the lines of the epilogue bodies and of their call sites in one source file."""
    src = open(path).read().splitlines()
    base = os.path.basename(path)
    out = {}

    def span(start, close):
        for k in range(start, len(src)):
            if re.match(close, src[k]):
                return range(start + 1, k + 2)
        raise ValueError("no end of the body at %s:%d" % (base, start + 1))

    for k, ln in enumerate(src):
        if base == "tcx_first.cuh":
            for name, body in (("l1_epilogue", "L1"), ("l2_epilogue", "L2")):
                if re.search(r"auto %s = \[&\]" % name, ln):
                    ind = len(ln) - len(ln.lstrip())
                    out.update({(base, i): body for i in span(k, r"^ {%d}};" % ind)})
                elif name + "(" in ln:
                    out[(base, k + 1)] = body
            if "xconv_block_epilogue<X3" in ln:
                out[(base, k + 1)] = "L3"
        elif base == "tcx_conv.cuh" and re.search(r"void xconv_block_epilogue\(", ln):
            out.update({(base, i): "L3" for i in span(k, r"^}")})
    return out


_BODIES = {}


def region_of(f, line):
    """Body a (file, line) location belongs to: L1 / L2 / L3, "other" for the rest of tcx_first.cuh, None for a helper's line."""
    base = os.path.basename(f)
    if base not in ("tcx_first.cuh", "tcx_conv.cuh"):
        return None
    if f not in _BODIES:
        _BODIES[f] = body_lines(f)
    r = _BODIES[f].get((base, line))
    return r if r is not None or base == "tcx_conv.cuh" else "other"


def outputs_per_thread(c1, cout, l3):
    """fp32 output values per consumer thread, summed over the unrolled copies of each body (8 layer-1 and 8 layer-2 blocks per
    warpgroup, 2 layer-3 blocks)."""
    return {"L1": 8 * c1 // 2, "L2": 8 * cout // 2, "L3": 2 * (2 * cout) // 2 if l3 else 0}


def count(sass, mangled):
    text = sass.split("\n.text._ZN2ag3tcx16tcx_first_kernelILi" + mangled, 1)[1]
    text = text.split("\n\t.section", 1)[0]
    where = {}
    cur = "other"
    counts = collections.defaultdict(collections.Counter)
    for ln in text.splitlines():
        m = ANN.search(ln)
        if m:
            f, line, pf, pline = m.group(1), int(m.group(2)), m.group(3), m.group(4)
            r = region_of(f, line)
            if r is None and pf is not None:
                r = region_of(pf, int(pline))
                if r is None:
                    r = where.get((os.path.basename(pf), int(pline)))
            if r is not None:
                where[(os.path.basename(f), line)] = r
                cur = r
            continue
        m = INS.search(ln)
        if m and m.group(1) not in ISSUE:
            counts[cur][m.group(1)] += 1
    return counts


def main():
    obj = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "affnet_b200", "csrc", "obj", "nets_tcx.o")
    with tempfile.TemporaryDirectory() as td:
        subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=td, check=True, capture_output=True)
        cubin = [f for f in os.listdir(td) if f.endswith(".cubin")][0]
        sass = subprocess.run(["nvdisasm", "-gi", "-c", os.path.join(td, cubin)], check=True, capture_output=True, text=True).stdout
    print("| instantiation | body | all | " + " | ".join(c for c, _ in CLASSES) + " | other |")
    print("|---|---|---|" + "---|" * (len(CLASSES) + 1))
    for name, mangled in INSTS:
        c1, cout, l3 = int(mangled[:2]), int(mangled[5:7]), int(mangled[-2])
        counts = count(sass, mangled)
        outs = outputs_per_thread(c1, cout, l3)
        for body in ("L1", "L2", "L3"):
            if not outs[body]:
                continue
            cnt = counts[body]
            total = sum(cnt.values())
            cells = []
            seen = 0
            for _, ops in CLASSES:
                k = sum(cnt[o] for o in ops)
                seen += k
                cells.append("%.2f" % (k / outs[body]))
            print("| %s | %s | %.2f (%d) | %s | %.2f |" % (name, body, total / outs[body], total, " | ".join(cells), (total - seen) / outs[body]))


if __name__ == "__main__":
    main()
