"""Instruction budget of the integer-ratio TMA resample kernel, read from the compiler's output (no GPU needed).

Compiles smelter_b200/csrc/kernels.cu alone with the library's nvcc flags into a temporary cubin and prints, for every
k_resample_tma3<S, SRC, FULL, MAT>: registers, spill stores / loads (ptxas -v), the kernel's SASS instruction count, and the
instruction count of the phase-A row loop (one warp, one source row: fetch, K1/K2, decode, horizontal pass, ring
store) by opcode.  The row loop is the backward-branch loop of the kernel that holds the SHFL.UP of the horizontal pass.
Then the same-ratio vertical pass of one step (one warp, two output rows): it is unrolled, so it is the branch-free run
of instructions outside the row loop with the most wide ring loads (LDS.64 / LDS.128); its FFMA and loads are printed, and
the ring rows they cover (3 * 8 / S floats per lane and ring row).

    python tools/tma3_sass_budget.py                  # the tree's kernels.cu
    python tools/tma3_sass_budget.py --csrc DIR       # another copy of smelter_b200/csrc, e.g. a parent commit's
    python tools/tma3_sass_budget.py --all            # also registers, spills and SASS count of every other kernel
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smelter_b200 import build as libbuild  # noqa: E402

_INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")
_FUNC = re.compile(r"^\s*Function : (\S+)")
_ENTRY = re.compile(r"Compiling entry function '(\S+)'")
_SPILL = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
_REGS = re.compile(r"Used (\d+) registers")


def compile_cubin(csrc, out_dir):
    """kernels.cu -> cubin with the library's code-generation flags; returns (sass text, ptxas -v text)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f for f in libbuild.NVCC_FLAGS if f != "-shared"]
    # host-compiler options do not change device code; -Xcompiler and its argument are dropped together
    keep = []
    skip = False
    for f in flags:
        if skip:
            skip = False
            continue
        if f == "-Xcompiler":
            skip = True
            continue
        keep.append(f)
    cubin = os.path.join(out_dir, "kernels.cubin")
    cmd = [nvcc] + keep + ["-Xptxas", "-v", "-cubin", "-o", cubin, os.path.join(csrc, "kernels.cu")]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout + p.stderr)
        raise SystemExit(f"nvcc failed ({p.returncode})")
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", cubin], capture_output=True,
                          text=True, check=True).stdout
    return sass, p.stdout + p.stderr


def parse_ptxas(text):
    """mangled name -> (registers, spill store bytes, spill load bytes)"""
    res, cur, spill = {}, None, (0, 0)
    for line in text.splitlines():
        m = _ENTRY.search(line)
        if m:
            cur, spill = m.group(1), (0, 0)
            continue
        m = _SPILL.search(line)
        if m and cur:
            spill = (int(m.group(1)), int(m.group(2)))
        m = _REGS.search(line)
        if m and cur:
            res[cur] = (int(m.group(1)),) + spill
            cur = None
    return res


def parse_sass(text):
    """mangled name -> [(address, opcode, operands)], the NOP padding after the final EXIT / BRA dropped"""
    funcs, cur = {}, None
    for line in text.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = _INSN.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(3), m.group(4).strip()))
    for name, ins in funcs.items():
        while ins and ins[-1][1] == "NOP":
            ins.pop()
    return funcs


def row_loop(ins):
    """the instructions of the smallest backward-branch loop that contains a SHFL.UP"""
    best = None
    for i, (addr, op, args) in enumerate(ins):
        if not op.startswith("BRA"):
            continue
        m = re.search(r"0x([0-9a-f]+)\s*$", args)
        if not m:
            continue
        tgt = int(m.group(1), 16)
        if tgt >= addr:
            continue
        body = [x for x in ins if tgt <= x[0] <= addr]
        if any(x[1].startswith("SHFL.UP") for x in body) and (best is None or len(body) < len(best)):
            best = body
    return best or []


def vertical_pass(ins, loop):
    """the branch-free run outside the row loop with the most LDS.64 / LDS.128 (the unrolled same-ratio vertical pass)"""
    inside = {x[0] for x in loop}
    targets = set()
    for _, op, args in ins:
        if op.startswith(("BRA", "BSSY")):
            m = re.search(r"0x([0-9a-f]+)\s*$", args)
            if m:
                targets.add(int(m.group(1), 16))
    blocks, cur = [], []
    for x in ins:
        if x[0] in targets and cur:
            blocks.append(cur)
            cur = []
        cur.append(x)
        if x[1].startswith(("BRA", "EXIT", "RET", "BRX")):
            blocks.append(cur)
            cur = []
    blocks.append(cur)

    def wide(b):
        return sum(1 for x in b if x[1].startswith(("LDS.64", "LDS.128")))
    return max((b for b in blocks if b and b[0][0] not in inside), key=wide, default=[])


def demangle_tma3(name):
    m = re.search(r"k_resample_tma3ILi(\d)ELi(\d)ELb(\d)E(?:Li(\d)E)?", name)   # kernels without MAT are BT.709
    return tuple(int(g or 0) for g in m.groups()) if m else None


def short_names(names, cuobjdump_dir):
    """mangled -> readable kernel names (cu++filt, namespaces and parameter lists dropped)"""
    out = subprocess.run([os.path.join(cuobjdump_dir, "cu++filt")], input="\n".join(names), capture_output=True, text=True,
                         check=True).stdout.splitlines()
    res = {}
    for n, d in zip(names, out):
        d = d[:d.rindex("(")] if "(" in d else d
        d = re.sub(r"^(void )?(\w+::)*", "", d)
        res[n] = re.sub(r"\(int\)", "", d).replace(" ", "")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--csrc", default=os.path.join(ROOT, "smelter_b200", "csrc"), help="directory holding kernels.cu")
    ap.add_argument("--all", action="store_true", help="list every kernel's registers, spills and SASS count")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory(prefix="tma3_sass_") as tmp:
        sass, ptxas = compile_cubin(os.path.abspath(a.csrc), tmp)
    regs = parse_ptxas(ptxas)
    funcs = parse_sass(sass)
    tma3 = sorted((demangle_tma3(n), n) for n in funcs if demangle_tma3(n))
    for (S, SRC, FULL, MAT), name in tma3:
        r, st, ld = regs.get(name, (0, 0, 0))
        loop = row_loop(funcs[name])
        print(f"k_resample_tma3<{S},{SRC},{FULL},{MAT}>: {r} registers, spill {st}/{ld} B, {len(funcs[name])} SASS; "
              f"phase-A row loop {len(loop)} instructions")
        ops = collections.Counter(op for _, op, _ in loop)
        const = sum(n for op, n in ops.items() if op.startswith(("ULDC", "LDC")))
        moves = sum(n for op, n in ops.items() if op == "MOV" or op.startswith("IMAD.MOV"))
        print(f"  constant loads {const}, register moves {moves}")
        line = []
        for op, n in sorted(ops.items(), key=lambda kv: (-kv[1], kv[0])):
            line.append(f"{op} {n}")
        for i in range(0, len(line), 8):
            print("  " + ", ".join(line[i:i + 8]))
        vp = collections.Counter(op.split(".reuse")[0] for _, op, _ in vertical_pass(funcs[name], loop))
        l64 = sum(n for op, n in vp.items() if op.startswith("LDS.64"))
        l128 = sum(n for op, n in vp.items() if op.startswith("LDS.128"))
        ffma = sum(n for op, n in vp.items() if op.startswith("FFMA"))
        print(f"  same-ratio vertical pass, one warp and step: FFMA {ffma}, LDS.64 {l64}, LDS.128 {l128}: "
              f"{(2 * l64 + 4 * l128) * S // 24} ring rows")
    if a.all:
        print()
        nvcc_dir = os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))
        short = short_names(sorted(funcs), nvcc_dir)
        for name in sorted(funcs, key=lambda n: short[n]):
            r, st, ld = regs.get(name, (0, 0, 0))
            print(f"{short[name]:32s} {r:4d} regs  spill {st:3d}/{ld:3d} B  {len(funcs[name]):6d} SASS")


if __name__ == "__main__":
    main()
