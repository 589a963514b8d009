"""The dense instantiations of the from-logits kernels must not change when the compact layout is added: compare the
SASS of every dense k_lse_pairs / k_expand_logits of two builds, instruction for instruction (no GPU needed).

    python tools/logits_sass_diff.py OLD/librnnt_b200.so NEW/librnnt_b200.so

OLD may predate the kernels' COMPACT template flag; NEW's COMPACT=false instantiations are matched to OLD's functions
of the same element type and vector width.  Exits 1 when any dense function differs or has no counterpart."""
import re
import subprocess
import sys


def funcs(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    fs, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            fs[fn] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if fn and m:
            fs[fn].append(m.group(1).strip())
    return fs


def key(name):
    """(kernel, mangled template arguments) of a from-logits kernel, else None."""
    m = re.match(r"_ZN4rnnt(1[15])(k_lse_pairs|k_expand_logits)I(.*?)EEEv", name)
    return (m.group(2), m.group(3)) if m else None


def main():
    old, new = funcs(sys.argv[1]), funcs(sys.argv[2])
    okeys = {key(n): n for n in old if key(n)}
    n_same = n_diff = 0
    for n, ins in new.items():
        k = key(n)
        if not k:
            continue
        kind, targs = k
        if targs.endswith("ELb1"):
            continue                                    # compact instantiation: new
        assert targs.endswith("ELb0"), n
        ok_targs = targs[:-len("ELb0")]
        match = okeys.get((kind, ok_targs))
        if match is None:
            print("no counterpart in OLD for", n)
            n_diff += 1
            continue
        same = old[match] == ins
        n_same += same
        n_diff += not same
        print("%-5s %-60s %d instructions" % ("same" if same else "DIFF", kind + "<" + ok_targs + ">", len(ins)))
    print("dense instantiations identical: %d, different: %d" % (n_same, n_diff))
    sys.exit(1 if n_diff else 0)


if __name__ == "__main__":
    main()
