#!/usr/bin/env python
"""Per-column instruction mix of ed_small_kernel's four-column fast block, read from `cuobjdump -sass` of the built library.

For each instantiation ed_small_kernel<NW, MODE, WANT_END> the SASS is split into basic blocks (labels and branches end a block).
The fast block is the one with the most LDS: the four Myers columns of one target word whose bytes are all ACGT, with their Peq loads
and the decode of the word. Its counts are divided by four and grouped by the pipe an instruction issues to:

  alu   integer ALU pipe (16 lanes per SMSP: a warp instruction holds it for 2 cycles): LOP3, SHF, IADD3, VIMNMX*, LEA, PRMT, ISETP, SEL, ...
  fma   FMA pipe: IMAD* (also the IMAD.MOV / IMAD.SHL forms ptxas uses to offload moves and shifts)
  lds   shared-memory loads
  vshr  variable-amount right shifts (SHF.R with a register shift amount) among the alu instructions

pair_report() gives the same mix for ed_pair_kernel<NW> per job-column (its fast block runs four columns of two jobs), pack_report() for
ed_pack_kernel<W, WA> (four columns of one W-word column that holds two jobs), and small_prologues() / prologue_alu() count the ALU
instructions of the job load and Peq build (up to the function's last STS).

Usage: python tools/sass_mix.py [LIB] [--json]   (LIB defaults to the in-tree delly_b200/libdelly_b200.so)
"""
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {0: "NW", 1: "SHW", 2: "HW"}
ALU = ("LOP3", "LOP", "SHF", "IADD3", "VIMNMX", "VIMNMX3", "IMNMX", "LEA", "PRMT", "ISETP", "SEL", "IABS", "BMSK", "SGXT", "FLO", "POPC",
       "PLOP3", "P2R", "R2P")
BRANCH = ("BRA", "EXIT", "RET", "CALL", "BRX", "JMP", "JMX")
INSN = re.compile(r"/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)\s*([^;]*);")
KERNEL = re.compile(r"ed_small_kernelILi(\d)ELi(\d)ELb(\d)E")
PAIR_KERNEL = re.compile(r"ed_pair_kernelILi(\d)E")
PACK_KERNEL = re.compile(r"ed_pack_kernelILi(\d)ELi(\d)E")


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def functions(sass):
    """{mangled name: [SASS lines]} of every function in the dump."""
    out, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            out[name].append(line)
    return out


def blocks(lines):
    """Basic blocks as lists of (opcode, operands)."""
    cur, res = [], []
    for line in lines:
        if re.match(r"\s*\.L_\w+:", line):
            if cur:
                res.append(cur)
            cur = []
            continue
        m = INSN.search(line)
        if not m:
            continue
        cur.append((m.group(2), m.group(3)))
        if m.group(2).split(".")[0] in BRANCH:
            res.append(cur)
            cur = []
    if cur:
        res.append(cur)
    return res


def mix(lines):
    """Per-column counts of the fast block of one ed_small_kernel instantiation."""
    fast = max(blocks(lines), key=lambda b: sum(op.startswith("LDS") for op, _ in b))
    c = {"alu": 0, "fma": 0, "lds": 0, "other": 0, "vshr": 0}
    ops = {}
    for op, args in fast:
        base = op.split(".")[0]
        ops[base] = ops.get(base, 0) + 1
        if base == "LDS":
            c["lds"] += 1
        elif base == "IMAD":
            c["fma"] += 1
        elif base in ALU:
            c["alu"] += 1
            # SHF.R.* with a register (not an immediate) shift amount: the third source operand
            if base == "SHF" and ".R." in op + "." and re.match(r"\S+,\s*\S+,\s*R\d+(\.reuse)?,", args):
                c["vshr"] += 1
        elif base not in BRANCH:
            c["other"] += 1
    res = {k: v / 4 for k, v in c.items()}
    res["ops"] = {k: v / 4 for k, v in sorted(ops.items())}
    return res


def prologue_alu(lines):
    """Integer-ALU instructions from the start of a function through its last shared-memory store: for ed_small_kernel and ed_pair_kernel
    the job load and the Peq build (with the set-up of the out-of-line calls that build words holding a byte outside ACGT)."""
    ops = [m.group(2) for m in map(INSN.search, lines) if m]
    last = max(i for i, op in enumerate(ops) if op.startswith("STS"))
    return sum(op.split(".")[0] in ALU for op in ops[:last + 1])


def _per_job(lines):
    """mix() of a kernel whose column steps advance two jobs, per job-column, with "prologue_alu"."""
    r = mix(lines)
    r = {k: (v / 2 if k != "ops" else {o: n / 2 for o, n in v.items()}) for k, v in r.items()}
    r["prologue_alu"] = prologue_alu(lines)
    return r


def pair_report(lib):
    """{"NW=n": mix} of the fast block of ed_pair_kernel<n>, per job-column (the block runs four columns of two jobs), with "prologue_alu"."""
    res = {}
    for name, lines in functions(_sass(lib)).items():
        m = PAIR_KERNEL.search(name)
        if m:
            res[f"NW={m.group(1)}"] = _per_job(lines)
    return dict(sorted(res.items()))


def pack_report(lib):
    """{"W=w WA=a": mix} of the fast block of ed_pack_kernel<w, a>, per job-column (the block runs four columns of one packed column that
    holds two jobs), with "prologue_alu"."""
    res = {}
    for name, lines in functions(_sass(lib)).items():
        m = PACK_KERNEL.search(name)
        if m:
            res[f"W={m.group(1)} WA={m.group(2)}"] = _per_job(lines)
    return dict(sorted(res.items()))


def small_prologues(lib):
    """{"NW=n MODE[ end]": prologue_alu} of every ed_small_kernel instantiation."""
    res = {}
    for name, lines in functions(_sass(lib)).items():
        m = KERNEL.search(name)
        if m:
            nw, mode, end = int(m.group(1)), int(m.group(2)), int(m.group(3))
            res[f"NW={nw} {MODES[mode]}{' end' if end else ''}"] = prologue_alu(lines)
    return dict(sorted(res.items()))


def _sass(lib):
    return subprocess.run([cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout


def report(lib):
    sass = _sass(lib)
    res = {}
    for name, lines in functions(sass).items():
        m = KERNEL.search(name)
        if m:
            nw, mode, end = int(m.group(1)), int(m.group(2)), int(m.group(3))
            res[f"NW={nw} {MODES[mode]}{' end' if end else ''}"] = mix(lines)
    return dict(sorted(res.items()))


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    lib = args[0] if args else os.path.join(ROOT, "delly_b200", "libdelly_b200.so")
    res = report(lib)
    pairs = {f"pair {k}": v for k, v in pair_report(lib).items()}
    packs = {f"pack {k}": v for k, v in pack_report(lib).items()}
    if "--json" in sys.argv:
        print(json.dumps({**res, **pairs, **packs}))
        return
    print(f"{'kernel':<16} {'alu':>6} {'fma':>6} {'lds':>5} {'other':>6} {'vshr':>5}   alu opcodes per column")
    for k, v in res.items():
        alu_ops = " ".join(f"{o}:{n:g}" for o, n in v["ops"].items() if o in ALU)
        print(f"{k:<16} {v['alu']:6.2f} {v['fma']:6.2f} {v['lds']:5.2f} {v['other']:6.2f} {v['vshr']:5.2f}   {alu_ops}")
    print(f"\n{'two-job kernel':<16} {'alu':>6} {'fma':>6} {'lds':>5} {'other':>6} {'vshr':>5} {'prologue':>8}   alu opcodes per job-column")
    for k, v in {**pairs, **packs}.items():
        alu_ops = " ".join(f"{o}:{n:g}" for o, n in v["ops"].items() if o in ALU)
        print(f"{k:<16} {v['alu']:6.2f} {v['fma']:6.2f} {v['lds']:5.2f} {v['other']:6.2f} {v['vshr']:5.2f} {v['prologue_alu']:8d}   {alu_ops}")


if __name__ == "__main__":
    main()
