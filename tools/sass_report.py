#!/usr/bin/env python
"""Static evidence from the built library, no GPU needed: per-kernel registers / stack / shared memory
(``cuobjdump -res-usage``) and the SASS mnemonics that matter for this path (``cuobjdump -sass``): the NVSwitch multicast
instructions (LDGMC / multimem stores), system-scope release/acquire traffic, TMA bulk copies, local-memory spills.

    mkdir -p tool_out && python tools/sass_report.py > tool_out/sass_report.md

``--digest [LIB]`` prints one line per kernel instead, ``<demangled name> <sha256 of its SASS>``, for LIB (default: the
in-tree library).  Two builds whose digests are equal have identical kernels, so a refactor of the device code can be
checked against the library built from its parent commit:

    diff <(python tools/sass_report.py --digest parent.so) <(python tools/sass_report.py --digest)
"""
import collections
import hashlib
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "torchx_b200", "lib", "libb200ddp.so")

INTERESTING = ("LDGMC", "MULTIMEM", "RED", "UBLKCP", "SYNCS", "MEMBAR", "CCTL", "F2FP", "STL", "LDL", "BAR", "ERRBAR", "HMMA", "UTC", "FENCE", "ATOM")
MODES = {0: "f32 bucket, bf16 wire", 1: "f32 bucket, f32 wire", 2: "bf16 bucket", 3: "f32 bucket, fp16 wire", 4: "fp16 bucket"}


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    clean = []
    for d in out:
        d = re.sub(r"\(anonymous namespace\)::", "", d)
        d = re.sub(r"^void ", "", d)
        d = re.sub(r"\(.*$", "", d)  # drop the parameter list
        clean.append(d)
    return dict(zip(names, clean))


def digest(lib: str) -> None:
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    body = collections.defaultdict(list)
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
        elif cur and line.lstrip().startswith("/*"):  # an instruction or the second half of its encoding
            body[cur].append(line.strip())
    names = demangle(sorted(body))
    # the anonymous namespace's hash (in mangled names) changes with any edit to the translation unit
    anon = re.compile(r"_GLOBAL__N__[0-9a-f]+_")
    for name, mangled in sorted((anon.sub("_GLOBAL__N__", names[k]), k) for k in body):
        print(name, hashlib.sha256(anon.sub("_GLOBAL__N__", "\n".join(body[mangled])).encode()).hexdigest())


def main() -> None:
    if "-h" in sys.argv or "--help" in sys.argv:
        print(__doc__)
        return
    if "--digest" in sys.argv:
        rest = sys.argv[sys.argv.index("--digest") + 1:]
        return digest(rest[0] if rest else LIB)
    if not os.path.isfile(LIB):
        raise SystemExit(f"{LIB} is not built: python -c 'import __graft_entry__ as g; g.build()'")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            usage[cur] = {k: int(v) for k, v in re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", line)}
            cur = None
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    counts = collections.defaultdict(collections.Counter)
    n_instr = collections.Counter()
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z][A-Z0-9_.]*)", line)
        if cur and m:
            op = m.group(1)
            n_instr[cur] += 1
            if op.split(".")[0].startswith(INTERESTING) or ".SYS" in op or ".256" in op or ".128" in op:
                counts[cur][op] += 1
    names = demangle(sorted(usage))
    print("# Static evidence from `torchx_b200/lib/libb200ddp.so` (sm_90a), produced by `tools/sass_report.py` (no GPU involved)\n")
    print(f"Kernels in the library: {len(usage)}.  Template arguments: `<MODE, W[, ALG]>`, MODE {MODES}; `k_pipe`'s ALG 0 = NVLS (multicast), 1 = P2P.\n")
    tc = sum(c for k in counts for op, c in counts[k].items() if op.startswith(("HMMA", "UTC")))
    print(f"Tensor-core instructions in the whole library (HMMA / UTC*MMA): {tc} - the path is a bandwidth-bound reduction, by design.\n")
    print("## 1. Registers, stack (spills) and static shared memory per kernel\n")
    print("`STACK` > 0 means ptxas spilled; `STL`/`LDL` are the spill instructions themselves.  All kernels launch 512 threads, 1 CTA / SM"
          " (so the budget is 128 registers).\n")
    print("| kernel | REG | STACK B | SHARED B | SASS instr. | STL / LDL |")
    print("|---|---:|---:|---:|---:|---:|")
    spilled = []
    for mangled in sorted(usage, key=lambda k: names[k]):
        u, c = usage[mangled], counts[mangled]
        stl = sum(v for op, v in c.items() if op.startswith("STL"))
        ldl = sum(v for op, v in c.items() if op.startswith("LDL"))
        if u["STACK"] or stl or ldl:
            spilled.append(names[mangled])
        print(f"| `{names[mangled]}` | {u['REG']} | {u['STACK']} | {u['SHARED']} | {n_instr[mangled]} | {stl} / {ldl} |")
    print(f"\nKernels with any spill: {len(spilled)} of {len(usage)}" + (": " + ", ".join(f"`{s}`" for s in spilled) if spilled else "") + ".\n")
    print("## 2. Mnemonics per kernel family (the W=8 instances of the DDP configuration: f32 bucket, bf16 wire)\n")
    print("`LDGMC...RED/ADD` is `multimem.ld_reduce` (the switch adds the W copies and returns one vector), a `.STRONG.SYS` store to the multicast"
          " address is `multimem.st`; `MEMBAR.ALL.SYS` + `ST.STRONG.SYS` is the release of a flag, `LD.STRONG.SYS` + `CCTL.IVALL` the acquiring"
          " poll; `UBLKCP` is `cp.async.bulk` (TMA) with `SYNCS` its mbarrier; `F2FP.BF16` the fused fp32->bf16 cast.\n")
    print("| kernel | mnemonic: count |")
    print("|---|---|")
    shown = 0
    for mangled in sorted(usage, key=lambda k: names[k]):
        nm = names[mangled]
        if re.search(r"<0, 8(, \d)?>|<0>|k_barrier|k_broadcast", nm):
            body = ", ".join(f"{op}: {v}" for op, v in sorted(counts[mangled].items()) if not op.startswith(("BAR", "STL", "LDL")))
            print(f"| `{nm}` | {body} |")
            shown += 1
    mc = {names[k]: sum(v for op, v in counts[k].items() if op.startswith("LDGMC") or "MULTIMEM" in op) for k in usage}
    with_mc = sorted(k for k, v in mc.items() if v)
    print(f"\nKernels containing multicast-reduce loads (`LDGMC`): {len(with_mc)}: " + ", ".join(f"`{k}`" for k in with_mc) + ".")


if __name__ == "__main__":
    sys.exit(main())
