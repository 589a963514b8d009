"""Scheduling lint for the fused kernel's recurrence loop (no GPU needed; needs cuobjdump).

ptxas sometimes runs a lane's two exact-LSE chains one after the other instead of interleaved, which lengthens the
dependent chain of every anti-diagonal.  In a well-scheduled step the two MUFU.EX2 of the two chains are a few
instructions apart; serialised, they are ~40 apart.  Prints the distances for every k_fused<exact, *, C=2> kernel and
exits 1 if a loop step is serialised.

    python tools/sass_check.py [path/to/librnnt_b200.so]
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
    fn, ins, bad = None, [], 0
    funcs = {}
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            funcs[fn] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if fn and m:
            funcs[fn].append(m.group(1).strip())
    for fn, ins in funcs.items():
        if not re.search(r"k_fusedILi1ELi[01]ELi2E", fn):      # dense exact flavour, two columns per lane (cfg 2)
            continue
        # the loop step: from a SHFL.UP by 1 to the next STS
        dist = []
        i = 0
        while i < len(ins):
            if ins[i].startswith("SHFL.UP") and "0x1, RZ" in ins[i]:
                mufu = []
                j = i + 1
                while j < len(ins) and not ins[j].startswith("SHFL.UP") and j - i < 200:
                    if "MUFU.EX2" in ins[j]:
                        mufu.append(j)
                    j += 1
                if len(mufu) >= 2:
                    dist.append(mufu[1] - mufu[0])
                i = j
            else:
                i += 1
        ok = sum(d > 20 for d in dist) <= 1          # the step before the back-edge is allowed to be serialised
        bad += not ok
        print("%-60s MUFU.EX2 distances per step: %s  %s" % (fn[:60], dist, "ok" if ok else "SERIALISED"))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
