"""Summarise an nvcc -Xptxas -v log: one line per kernel (demangled template args, registers, spills, smem)."""
import re
import subprocess
import sys


def main(path, pat=""):
    txt = open(path).read()
    rows = []
    for m in re.finditer(r"Compiling entry function '(\S+)' for 'sm_90a'\n(?:.*\n)*?.*Used (\d+) registers(.*)", txt):
        name, regs, rest = m.group(1), int(m.group(2)), m.group(3)
        rows.append((name, regs, rest))
    if not rows:
        return
    dem = subprocess.run(["c++filt"] + [r[0] for r in rows], capture_output=True, text=True).stdout.splitlines()
    spills = dict()
    for m in re.finditer(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores", txt):
        spills[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    for (name, regs, rest), d in zip(rows, dem):
        short = re.sub(r"\(.*", "", d).replace("llmlb::", "").replace("void ", "")
        if pat and pat not in short:
            continue
        sp = spills.get(name, (0, 0))
        sm = re.search(r"(\d+) bytes smem", rest)
        print("%-70s regs=%3d stack=%d spill=%d smem=%s" % (short, regs, sp[0], sp[1], sm.group(1) if sm else "0"))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "")
