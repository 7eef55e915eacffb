#!/usr/bin/env python3
"""Instruction census of the CWBVH8 node step, from the SASS of a compiled object or library (CPU only, needs cuobjdump on PATH or in /usr/local/cuda/bin).

    python scripts/sass_census.py rtxpt_b200/csrc/_build/fast/kernels.o 'k_trace_closestILb0ELi4ELb1'
    python scripts/sass_census.py rtxpt_b200/csrc/_build/fast/kernels.o k_trace --ptxas-log rtxpt_b200/csrc/_build/fast/kernels.ptxas.log

For every kernel whose mangled name contains the pattern it cuts the node step of Traverser::run (traverse.cuh) - from the group of five LDG.E.128.CONSTANT that loads the 80-byte
node to the first LDL after it, the pop of the traversal stack - and counts the instructions per issue pipe: `fma` (FP32 add / multiply / FMA, 128 results per clock per SM in
the arithmetic-throughput table of the CUDA programming guide for compute capability 9.0, and the integer multiply-add that shares that pipe), `alu` (FP32 and integer min / max /
compare, integer add, logic, shift, select, permute: 64), `xu` (conversions, special functions, population count).  The assignment of an opcode to a class is this script's
reading of that table, and the count is what one lane issues on one visit of the straight-line node step - not a measurement: no counter of the GPU is read.
With --ptxas-log the registers, stack frame and spills `-Xptxas -v` reported for the same kernels are printed beside the counts."""
import argparse
import collections
import os
import re
import shutil
import subprocess
import sys

PIPES = collections.OrderedDict([
    ("fma", ("FFMA", "FMUL", "FADD", "IMAD")),
    ("alu", ("FMNMX", "VIMNMX", "VIMNMX3", "LOP3", "SHF", "SEL", "FSEL", "FSETP", "ISETP", "PRMT", "IADD3", "VIADD", "LEA", "MOV", "PLOP3", "BMSK", "SGXT", "IABS", "VABSDIFF", "FCHK")),
    ("xu", ("I2F", "I2FP", "F2I", "F2F", "MUFU", "POPC", "FLO", "BREV")),
])
NODE_LOAD = "LDG.E.128.CONSTANT"


def cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        sys.exit("cuobjdump not found")
    return exe


def functions(path):
    """{mangled name: [instruction text, ...]} of every kernel in the file."""
    text = subprocess.run([cuobjdump(), "-sass", path], check=True, capture_output=True, text=True).stdout
    out, cur = collections.OrderedDict(), None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur is not None:
            cur.append(m.group(1).strip())
    return out


def opcode(ins):
    parts = ins.split()
    op = parts[1] if parts[0].startswith("@") else parts[0]
    return op


def node_step(instructions):
    """The instructions from the first group of five node loads to the stack pop that follows it, or None."""
    loads = [i for i, ins in enumerate(instructions) if opcode(ins) == NODE_LOAD]
    for k in range(len(loads) - 4):
        if loads[k + 4] - loads[k] <= 16:
            first = loads[k]
            for j in range(loads[k + 4], len(instructions)):
                if opcode(instructions[j]).startswith("LDL"):
                    return instructions[first:j]
            return None
    return None


def census(region):
    by_pipe = collections.OrderedDict((p, collections.Counter()) for p in list(PIPES) + ["other"])
    for ins in region:
        op = opcode(ins)
        base = op.split(".")[0]
        for pipe, names in PIPES.items():
            if base in names:
                by_pipe[pipe][base] += 1
                break
        else:
            by_pipe["other"][base] += 1
    return by_pipe


def ptxas_resources(log):
    """{mangled name: 'NN registers, NN B stack, NN B spill stores, NN B spill loads'} from an `-Xptxas -v` log."""
    res, name, stack = {}, None, ""
    for line in open(log):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            stack = "%s B stack, %s B spill stores, %s B spill loads" % m.groups()
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            res[name] = "%s registers, %s" % (m.group(1), stack)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("binary", help="object file or shared library with sm_90a SASS")
    ap.add_argument("pattern", help="substring of the mangled kernel name, e.g. k_trace_closestILb0ELi4ELb1")
    ap.add_argument("--ptxas-log", help="the -Xptxas -v log of the same compilation (csrc/Makefile writes <unit>.ptxas.log)")
    args = ap.parse_args()
    resources = ptxas_resources(args.ptxas_log) if args.ptxas_log else {}
    found = 0
    for name, instructions in functions(args.binary).items():
        if args.pattern not in name:
            continue
        found += 1
        region = node_step(instructions)
        print(name + ("   [" + resources[name] + "]" if name in resources else ""))
        if region is None:
            print("  no node step found (five %s in a row, then an LDL)" % NODE_LOAD)
            continue
        c = census(region)
        print("  node step: %d instructions" % len(region))
        for pipe, counts in c.items():
            print("  %-5s %4d   %s" % (pipe, sum(counts.values()), ", ".join("%s %d" % kv for kv in counts.most_common())))
    if not found:
        sys.exit("no kernel name contains %r" % args.pattern)


if __name__ == "__main__":
    main()
