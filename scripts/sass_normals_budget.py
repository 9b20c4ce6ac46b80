"""Instruction budget of the 7x11 normals kernels from their SASS (no GPU needed).

Runs `cuobjdump -sass` on the object normals.cu was compiled to (delora_b200/build/normals.o after build.py, or the
object given as the first argument) and prints, for project_normals_7x11_kernel<3|4> and normals_7x11_kernel, the
length of every loop the compiler kept: the tap loop (one column of 2 x 7 pixel-taps per trip, 11 trips per thread)
and the Jacobi sweep loop (one per pixel of the thread's two, 3-4 trips each).  A loop is the address range from the
target of a backward branch to the branch; it is a tap column when it reads shared memory with LDS.128 and a Jacobi
sweep when it uses the MUFU unit.

    python scripts/sass_normals_budget.py [path/to/normals.o]
"""
import collections
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_OBJ = os.path.join(HERE, "..", "delora_b200", "build", "normals.o")
KERNELS = {"project_normals_7x11_kernelILi3E": "project_normals_7x11_kernel<3>",
           "project_normals_7x11_kernelILi4E": "project_normals_7x11_kernel<4>",
           "normals_7x11_kernel": "normals_7x11_kernel"}
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?);")
BRANCH = re.compile(r"^(?:@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(?:`\(\.L_x_\d+\)|0x([0-9a-f]+))")


def functions(sass):
    """{mangled name: [(address, instruction text)]} for every function in the cuobjdump listing."""
    out, cur = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = out.setdefault(line.split("Function :")[1].strip(), [])
            continue
        m = INSN.match(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2).strip()))
    return out


def loops(insns):
    """[(first address, last address, [instruction text])] for every backward branch."""
    addr_of = {a: i for i, (a, _) in enumerate(insns)}
    found = []
    for i, (a, text) in enumerate(insns):
        m = BRANCH.match(text)
        if not m or m.group(1) is None:
            continue
        target = int(m.group(1), 16)
        if target < a and target in addr_of:
            found.append((target, a, [t for _, t in insns[addr_of[target]:i + 1]]))
    return found


def opcode(text):
    text = re.sub(r"^@!?U?P\w+\s+", "", text)
    return text.split()[0] if text else ""


def main(argv):
    obj = argv[1] if len(argv) > 1 else DEFAULT_OBJ
    sass = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
    for mangled, insns in functions(sass).items():
        name = next((v for k, v in KERNELS.items() if k in mangled), None)
        if name is None:
            continue
        print(f"{name}: {len(insns)} instructions")
        for lo, hi, body in loops(insns):
            ops = collections.Counter(opcode(t).split(".")[0] for t in body)
            if any(opcode(t).startswith("LDS.128") for t in body):
                kind = "tap column"
            elif ops["MUFU"] >= 6:
                kind = "Jacobi sweep"
            else:
                continue
            top = ", ".join(f"{k} {v}" for k, v in ops.most_common(8))
            print(f"  {kind:12s} {len(body):4d} instructions  [{lo:#06x}, {hi:#06x}]  {top}")


if __name__ == "__main__":
    main(sys.argv)
