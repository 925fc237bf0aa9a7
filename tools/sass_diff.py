"""Dev tool: which kernels of two builds of libdsgd.so differ, instruction for instruction (cuobjdump -sass; addresses and
encodings ignored).  Used to show that adding template variants leaves the kernels that were verified on the GPU untouched.
    python tools/sass_diff.py old/libdsgd.so distributed_sgd_b200/libdsgd.so
A kernel that gained trailing template arguments 0 or false (e.g. `..., 0>` -> `..., 0, 0>`, `..., false>` ->
`..., false, false>`) is matched by its name prefix.  A kernel with no such counterpart is matched to every kernel of the
second build with the identical instruction list and reported as renamed; matching by body is many-to-one (two
instantiations can compile to the same instructions), so it is evidence of a rename, not a proof.
    --mask-params (before the paths): the body match ignores which kernel parameter an instruction reads (c[0x0][0x...]
    operands), so a kernel whose parameters moved by a slot is still reported as renamed.
    --mask-regs (before the paths): a kernel whose instructions differ only in register names (R, UR, P and UP registers;
    RZ, URZ, PT and UPT are kept) is reported as "registers only" rather than DIFFERENT; the body match ignores them too."""
import re
import subprocess
import sys


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    d, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            d[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(.*?)\s*/\*", line)
        if m and cur is not None:
            d[cur].append(m.group(1))
    return d


def main():
    flags = [f for f in ("--mask-params", "--mask-regs") if f in sys.argv[1:-2]]
    a, b = kernels(sys.argv[-2]), kernels(sys.argv[-1])
    regs = lambda i: re.sub(r"\b(U?[RP])\d+\b", r"\1#", i) if "--mask-regs" in flags else i
    params = lambda i: re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][param]", i) if "--mask-params" in flags else i
    key = lambda body: tuple(params(regs(i)) for i in body)
    by_body = {}
    for name, body in b.items():
        by_body.setdefault(key(body), []).append(name)
    differ = renamed = reg_only = 0
    for name, body in sorted(a.items()):
        extra = ("ELi0", "ELi0ELi0", "ELb0")
        cands = [name] if name in b else [n for n in (name.replace("EEEv", e + "EEEv", 1) for e in extra) if n in b]
        if not cands:
            same = by_body.get(key(body))
            if same:
                print("renamed:", name, "->", " | ".join(sorted(same)))
                renamed += 1
            else:
                print("only in the first build:", name)
                differ += 1
        elif body != b[cands[0]] and [regs(i) for i in body] == [regs(i) for i in b[cands[0]]]:
            print("registers only:", name, len(body), "instructions")
            reg_only += 1
        elif body != b[cands[0]]:
            print("DIFFERENT:", name, len(body), "->", len(b[cands[0]]), "instructions")
            differ += 1
    print(f"{len(a)} kernels in the first build, {len(b)} in the second, {renamed} renamed, "
          + (f"{reg_only} differ only in registers, " if "--mask-regs" in flags else "")
          + f"{differ} differ or are missing")
    return 1 if differ else 0


if __name__ == "__main__":
    raise SystemExit(main())
