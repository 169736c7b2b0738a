#!/usr/bin/env python
"""Instructions per Runge-Kutta stage of the fused 2xFP16 solve, counted in its SASS (no GPU needed).

    python scripts/stage_sass_count.py [--csrc DIR] [--kernel NAME] [--top N]

Compiles DIR/solve_tc.cu (default: this tree's torchcde_b200/csrc) for sm_90a with the library's flags and -Xptxas -v,
prints every cdeint_wgmma_kernel instantiation's registers and spill, then splits the stage loop of one instantiation
(default: the forward solve, cdeint_wgmma_kernel<false, false, false>) into three regions by address:
  * top: from the loop head to the first HGMMA (spline rows, dX/dt, the row scales, the A fragments, chunk 0's bias);
  * wgmma: from the first HGMMA to the last instruction that the line table attributes to wg::field (the products,
    the other chunks' bias, the contraction);
  * combination: the rest of the loop body (the Runge-Kutta combination of every method, the outputs, the loop control).
The stage loop is the innermost loop (a backward branch) that encloses every HGMMA.  A warp executes the top and wgmma
regions once per stage; the combination region holds every method's branch, of which a stage runs one."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo"]
FORWARD = "_ZN4tcde2tc19cdeint_wgmma_kernelILb0ELb0ELb0EEEvNS_8UmmaArgsE"

INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?);")
LINE = re.compile(r'//## File "([^"]+)", line (\d+)')
LABEL = re.compile(r"^(\.L_x_\d+):")
TARGET = re.compile(r"\bBRA 0x([0-9a-f]+)")
BRANCH = re.compile(r"\bBRA\b.*?\(?(\.L_x_\d+)\)?")


def compile_cubin(csrc, out_dir):
    cubin = os.path.join(out_dir, "solve_tc.cubin")
    proc = subprocess.run(["nvcc"] + FLAGS + ["-Xptxas", "-v", "-cubin", "-o", cubin, os.path.join(csrc, "solve_tc.cu")],
                          capture_output=True, text=True)
    if proc.returncode != 0:
        sys.exit(proc.stdout + proc.stderr)
    return cubin, proc.stderr


def resources(ptxas_log):
    """{kernel: (registers, spill stores, spill loads)} of the cdeint_wgmma_kernel instantiations."""
    res, name, spill = {}, None, (0, 0)
    for line in ptxas_log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spill = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name and "cdeint_wgmma_kernel" in name:
            res[name] = (int(m.group(1)),) + spill
    return res


def disassemble(cubin, kernel):
    """[(address, instruction text with branch targets as addresses, (file, line))] of one kernel."""
    text = subprocess.run(["nvdisasm", "-g", "-c", cubin], capture_output=True, text=True, check=True).stdout
    out, inside, where, labels, pending = [], False, (None, 0), {}, []
    for line in text.splitlines():
        if line.startswith("//-----") and ".text." in line:
            inside = (".text." + kernel + " ") in line + " "
            continue
        if not inside:
            continue
        m = LABEL.match(line)
        if m:
            pending.append(m.group(1))
            continue
        m = LINE.search(line)
        if m:
            where = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = INSN.match(line)
        if m:
            out.append((int(m.group(1), 16), m.group(2).strip(), where))
            labels.update((name, out[-1][0]) for name in pending)
            pending = []
    if not out:
        sys.exit("kernel {} not found in the cubin".format(kernel))
    return [(a, BRANCH.sub(lambda m: "BRA 0x{:x}".format(labels[m.group(1)]), s) if "BRA" in s else s, w)
            for a, s, w in out]


def field_lines(csrc):
    """The source lines of wg::field in solve_tc.cu: from its signature to the closing brace of its body."""
    src = open(os.path.join(csrc, "solve_tc.cu")).read().splitlines()
    start = next(i for i, s in enumerate(src) if re.search(r"\bvoid field\(", s)) + 1
    end = next(i for i in range(start, len(src)) if src[i].startswith("}")) + 1
    return start, end


def opcode(insn):
    body = re.sub(r"^@!?U?P\w+\s+", "", insn)
    return body.split()[0].split(".")[0]


def regions(insns, csrc):
    hgmma = [i for i, (_, s, _) in enumerate(insns) if "HGMMA" in s]
    if not hgmma:
        sys.exit("no HGMMA in the kernel")
    addr = [a for a, _, _ in insns]
    first, last = addr[hgmma[0]], addr[hgmma[-1]]
    loops = []
    for i, (a, s, _) in enumerate(insns):
        m = TARGET.search(s)
        if m and int(m.group(1), 16) <= first and a >= last:
            loops.append((int(m.group(1), 16), a))
    if not loops:
        sys.exit("no loop encloses the HGMMAs")
    head, tail = max(loops)                                      # the innermost: the latest head
    lo, hi = field_lines(csrc)
    body = [(a, s, w) for a, s, w in insns if head <= a <= tail]
    in_field = [a for a, s, w in body if w[0] == "solve_tc.cu" and lo <= w[1] <= hi]
    cut = max(in_field)
    return head, tail, {
        "top": [s for a, s, _ in body if a < first],
        "wgmma": [s for a, s, _ in body if first <= a <= cut],
        "combination": [s for a, s, _ in body if a > cut],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--csrc", default=os.path.join(ROOT, "torchcde_b200", "csrc"))
    ap.add_argument("--kernel", default=FORWARD)
    ap.add_argument("--top", type=int, default=12, help="opcodes listed per region")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        cubin, log = compile_cubin(args.csrc, tmp)
        print("registers, spill stores / loads (bytes):")
        for name, (regs, st, ld) in sorted(resources(log).items()):
            print("  {:64s} {:3d} registers, {} / {}".format(name, regs, st, ld))
        if "serialized" in log:
            print("ptxas: wgmma serialized")
        insns = disassemble(cubin, args.kernel)
    head, tail, parts = regions(insns, args.csrc)
    print("{}: stage loop 0x{:x}..0x{:x}, {} instructions".format(args.kernel, head, tail,
                                                                   sum(len(v) for v in parts.values())))
    for name, ops in parts.items():
        count = collections.Counter(opcode(s) for s in ops)
        uniform = sum(n for op, n in count.items() if op.startswith("U") or op == "R2UR")
        listed = ", ".join("{} {}".format(op, n) for op, n in count.most_common(args.top))
        print("  {:12s} {:4d} (uniform {:3d}): {}".format(name, len(ops), uniform, listed))


if __name__ == "__main__":
    main()
