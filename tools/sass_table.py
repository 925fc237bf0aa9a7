"""Static SASS facts per kernel of libdsgd.so (cuobjdump -sass / -res-usage): the mnemonics that prove TMA bulk copies,
mbarriers, fp64 reductions without a return value, system-scope LL stores, and the absence of tensor-core instructions.
    python tools/sass_table.py > sass_evidence.md"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "distributed_sgd_b200", "libdsgd.so")
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip().split("(")[0].replace("dsgd::", "").replace("void ", "")

COLS = [("UBLKCP (TMA)", r"\bUBLKCP"), ("SYNCS (mbarrier)", r"\bSYNCS"), ("REDG.F64", r"\bREDG\.E\.ADD\.F64"), ("all REDG", r"\bREDG"),
        ("ATOMG", r"\bATOMG"), ("LDG", r"\bLDG"), ("..STRONG.SYS ld/st", r"\b(LDG|STG|LD|ST)\.E(\.\d+)?\.STRONG\.SYS"), ("STG", r"\bSTG"),
        ("LDS", r"\bLDS"), ("fp64 math", r"\bD(ADD|MUL|FMA|SETP)"), ("SHFL", r"\bSHFL"), ("REDUX", r"\bREDUX"), ("BAR", r"\bBAR\."),
        ("MEMBAR/FENCE", r"\b(MEMBAR|FENCE)"), ("local ld/st (spills)", r"\b(LDL|STL)"), ("tensor (HMMA/UTC*MMA/…)", r"\b(HMMA|IMMA|DMMA|UTC\w*MMA|QGMMA)")]
counts, cur = collections.OrderedDict(), None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = demangle(m.group(1))
        counts[cur] = collections.Counter({"_n": 0})
        continue
    if cur is None or not re.match(r"\s+/\*[0-9a-f]{4,}\*/\s", line):
        continue
    counts[cur]["_n"] += 1
    for name, pat in COLS:
        if re.search(pat, line):
            counts[cur][name] += 1
usage = {}
for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res):
    usage[demangle(m.group(1))] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))

print("# SASS evidence (`cuobjdump -sass distributed_sgd_b200/libdsgd.so`, sm_90a, nvcc 12.9; `tools/sass_table.py`)\n")
print("What the mnemonics prove: `UBLKCP` = TMA bulk copy (`cp.async.bulk`), `SYNCS.*` = mbarrier (`arrive.expect_tx`,\n"
      "`try_wait`), `REDG.E.ADD.F64` = fp64 reduction at L2 WITHOUT a return value (gradient scatter; at `.SYS` scope the async peer-replica\n"
      "writes), `..STRONG.SYS` loads/stores = the LL words of the multi-GPU exchange (`st.relaxed.sys` / `ld.relaxed.sys`), `REDUX` = the\n"
      "warp or-reductions of the flat stream.  `ATOMG` = atomics WITH a return value: the streaming kernels' block tickets and nothing on\n"
      "the sync step's path (round 1 had 17 `ATOMG.E.ADD.F64 … RZ` there: nvcc's encoding of `atomicAdd(double*)` with an unused result; they\n"
      "are PTX `red` now).  No tensor-core instruction anywhere: this is a sparse dot-product path.  `<…, 1>` = multi-GPU instantiation of\n"
      "`k_sync_persistent`, `<…, 0>` the one-GPU loop.  Counts are static occurrences.\n")
print("| kernel | instr | " + " | ".join(n for n, _ in COLS) + " | regs | stack B | static smem B |")
print("|---|---|" + "---|" * (len(COLS) + 3))
for k, c in sorted(counts.items(), key=lambda kv: -kv[1]["_n"]):
    u = usage.get(k, ("?", "?", "?"))
    print(f"| `{k}` | {c['_n']} | " + " | ".join(str(c[n]) for n, _ in COLS) + f" | {u[0]} | {u[1]} | {u[2]} |")
