"""Write profiles/r<round>_sass_k_fused.txt from the built library (no GPU needed):

    python tools/sass_excerpts.py [round]

Mnemonic census of k_fused<exact, dense, C=2, float>, the bulk-copy (TMA engine) sites, one anti-diagonal step of a
recurrence loop (from one SHFL.UP to the next), the progress publication and the patch loop."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "warp_rnnt_b200", "lib", "librnnt_b200.so")
KERNEL = "_ZN4rnnt7k_fusedILi1ELi0ELi2EfEEvNS_9FusedArgsE"


def main():
    rnd = sys.argv[1] if len(sys.argv) > 1 else "2"
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    lines, on = [], False
    for ln in txt.splitlines():
        if "Function :" in ln:
            on = KERNEL in ln
            continue
        if on and re.match(r"\s+/\*[0-9a-f]{4,5}\*/", ln):
            lines.append(ln.rstrip())
    op = lambda ln: re.sub(r"^\s+/\*[0-9a-f]+\*/\s+(@!?U?P\d\s+)?", "", ln).split()[0].rstrip(";")
    census = collections.Counter()
    for ln in lines:
        o = op(ln)
        for key in ("UBLKCP", "SYNCS", "MUFU.EX2", "SHFL.UP", "SHFL.IDX", "LDS", "STS", "LDG", "STG", "ATOMS", "ATOMG",
                    "MEMBAR", "BAR", "NANOSLEEP", "FFMA", "FADD", "FMUL", "DMUL"):
            if o == key or o.startswith(key + "."):
                census[key] += 1
                break
    out = ["# SASS excerpts of rnnt::k_fused<exact, dense, C=2, float> (sm_90a), cuobjdump -sass of warp_rnnt_b200/lib/librnnt_b200.so",
           "# (regenerate with tools/sass_excerpts.py)  %d instructions in the kernel.  Mnemonic census:" % len(lines),
           "#   " + ", ".join("%s %d" % kv for kv in census.items()), ""]
    out.append("## bulk-copy (TMA engine) sites: row gather (global->shared, mbarrier completion) and zero-fill (shared->global)")
    out += [ln for ln in lines if op(ln).startswith(("UBLKCP", "SYNCS"))]
    # one step of the first recurrence loop: the span between two consecutive SHFL.UP that contains two MUFU.EX2
    idx = [i for i, ln in enumerate(lines) if op(ln).startswith("SHFL.UP")]
    step = None
    for a, b in zip(idx, idx[1:]):
        if sum(op(ln).startswith("MUFU.EX2") for ln in lines[a:b]) == 2 and b - a > 60:
            step = (a, b)
            break
    if step:
        out += ["", "## one anti-diagonal step of a recurrence loop (exact LSE, two columns per lane): from one SHFL.UP to the next, %d instructions" % (step[1] - step[0])]
        out += lines[step[0]:step[1] + 1]
    mem = [i for i, ln in enumerate(lines) if op(ln).startswith("MEMBAR")]
    loop_mem = [i for i in mem if step and i > step[0]]
    if loop_mem:
        i = loop_mem[0]
        out += ["", "## progress publication for the chasing warps (st.release.cta.shared = MEMBAR.ALL.CTA + STS), once per 8 steps"]
        out += lines[max(0, i - 5):i + 3]
    stg = [i for i, ln in enumerate(lines) if op(ln).startswith("STG") and i > (mem[-1] if mem else 0)]
    if stg:
        i = stg[0]
        out += ["", "## patch loop (after beta[0,0] is known): expf(x - beta00), scale, one STG per item, running cursor"]
        out += lines[max(0, i - 40):i + 10]
    path = os.path.join(ROOT, "profiles", "r%s_sass_k_fused.txt" % rnd)
    open(path, "w").write("\n".join(out) + "\n")
    print(path, len(out), "lines; step =", step and step[1] - step[0], "instructions")


if __name__ == "__main__":
    main()
