#!/usr/bin/env python3
"""SASS instructions of one kernel per named source region (runs without a GPU).

    scripts/sass_regions.py [BINARY] [--kernel SUBSTR] [--source FILE] [--regions name:first-last[:cold],...]
                            [--weight name=trips,...]

BINARY is a cubin, an object file or the built library (default xllm_service_b200/libxllm_ingest.so; cubins are taken
out of the latter two with cuobjdump).  The kernel is the first .text section whose mangled name holds SUBSTR
(default sp_express_kernelILb1, the narrow-id express kernel).  Regions are line ranges of --source: either given
with --regions, or read from the source's own markers

    // region: NAME          (a region runs to the line before the next marker)
    // region: NAME (cold)   (not executed in an all-hit step: left out of the hit-step sum)
    // region: end

An instruction belongs to the innermost frame of its inline chain (nvdisasm --print-line-info-inline) that lies in a
region: an unmarked helper's instructions count where the helper is called, a marked part of a helper on its own.
What lies in no region (the kernel's own loop, the out-of-line cooperative paths) is listed as "(none)".  The copies
of a step's code that the compiler keeps for a warp that reaches a vote or shuffle diverged (BRA.DIV targets, up to
the branch back) never run here, since the warp is converged at every one: they are listed apart.  --weight
multiplies a region's static count in the "executed" column: a loop that runs ~5 times per step is  scatter-loop=5 .
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARK = re.compile(r"//\s*region:\s*([A-Za-z0-9_+\-]+)\s*(\(cold\))?")
DIV = re.compile(r"BRA\.DIV .*`\((\.L_x_\d+)\)")
LABEL = re.compile(r"^(\.L_x_\d+):")
STUBS = "(diverged copies)"
FRAME = re.compile(r'//## File "([^"]+)", line (\d+)')
INSTR = re.compile(r"^\s+/\*[0-9a-f]+\*/\s+\S")


def marker_regions(source):
    """[(name, first, last, cold)] from the // region: markers of the source file."""
    out, cur = [], None
    with open(source) as f:
        lines = f.readlines()
    for no, text in enumerate(lines, 1):
        m = MARK.search(text)
        if not m:
            continue
        if cur:
            out.append((cur[0], cur[1], no - 1, cur[2]))
        cur = None if m.group(1) == "end" else (m.group(1), no, bool(m.group(2)))
    if cur:
        out.append((cur[0], cur[1], len(lines), cur[2]))
    return out


def cubins(binary, tmp):
    with open(binary, "rb") as f:
        head = f.read(20)
    if head[18:20] == b"\xbe\x00":   # e_machine EM_CUDA: already a cubin
        return [binary]
    subprocess.check_call(["cuobjdump", "-xelf", "all", os.path.abspath(binary)], cwd=tmp, stdout=subprocess.DEVNULL)
    return sorted(os.path.join(tmp, n) for n in os.listdir(tmp) if n.endswith(".cubin"))


def kernel_frames(cubin, substr):
    """(kernel name, [inline chain of every instruction, innermost frame first]) or None."""
    sass = subprocess.run(["nvdisasm", "--print-line-info-inline", cubin], check=True, capture_output=True,
                          text=True).stdout
    name, chains, chain, fresh, in_stub = None, [], [], True, False
    targets = set(DIV.findall(sass))
    for line in sass.splitlines():
        if line.startswith(".text."):
            if name:
                break
            if substr in line:
                name = line[len(".text."):].rstrip(":")
            continue
        if not name:
            continue
        if line.lstrip().startswith(".section"):
            break
        m = FRAME.search(line)
        if m:
            if fresh:
                chain, fresh = [], False
            chain.append((m.group(1), int(m.group(2))))
        elif LABEL.match(line):
            in_stub = in_stub or LABEL.match(line).group(1) in targets
        elif INSTR.match(line):
            chains.append(STUBS if in_stub else tuple(chain))
            fresh = True
            if in_stub and re.match(r"^\s+/\*[0-9a-f]+\*/\s+BRA ", line):
                in_stub = False
    return (name, chains) if name else None


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("binary", nargs="?", default=os.path.join(ROOT, "xllm_service_b200", "libxllm_ingest.so"))
    ap.add_argument("--kernel", default="sp_express_kernelILb1")
    ap.add_argument("--source", default=os.path.join(ROOT, "xllm_service_b200", "csrc", "sp_encode.cu"))
    ap.add_argument("--regions", default="")
    ap.add_argument("--weight", default="")
    a = ap.parse_args()
    if a.regions:
        regions = []
        for r in a.regions.split(","):
            name, span, *cold = r.split(":")
            first, last = span.split("-")
            regions.append((name, int(first), int(last), cold == ["cold"]))
    else:
        regions = marker_regions(a.source)
    if not regions:
        sys.exit("no regions: give --regions or mark the source with // region: comments")
    weight = {k: float(v) for k, v in (w.split("=") for w in a.weight.split(",") if w)}
    src = os.path.basename(a.source)

    def region_of(chain):
        if chain == STUBS:
            return STUBS
        for f, no in chain:                     # innermost frame first
            if os.path.basename(f) == src:
                for name, first, last, _ in regions:
                    if first <= no <= last:
                        return name
        return "(none)"

    with tempfile.TemporaryDirectory() as tmp:
        found = None
        for c in cubins(a.binary, tmp):
            found = kernel_frames(c, a.kernel)
            if found:
                break
    if not found:
        sys.exit("no kernel with %r in its name in %s" % (a.kernel, a.binary))
    name, chains = found
    count = collections.Counter(region_of(c) for c in chains)
    print("%s: %d instructions" % (name, len(chains)))
    print("%-22s %8s %9s" % ("region", "static", "executed"))
    hot_static, hot_exec = 0, 0.0
    for rname, first, last, cold in regions:
        n = count.get(rname, 0)
        if cold:
            print("%-22s %8d %9s   lines %d-%d" % (rname, n, "cold", first, last))
            continue
        e = n * weight.get(rname, 1.0)
        hot_static += n
        hot_exec += e
        print("%-22s %8d %9.0f   lines %d-%d" % (rname, n, e, first, last))
    for other in ("(none)", STUBS):
        print("%-22s %8d %9s" % (other, count.get(other, 0), "-"))
    print("%-22s %8d %9.0f" % ("hit step", hot_static, hot_exec))


if __name__ == "__main__":
    main()
