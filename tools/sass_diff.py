"""Compare the SASS of every function of two builds of the library, by name (no GPU needed).  A change that touches
only host code must leave every function identical.

    python tools/sass_diff.py OLD/librnnt_b200.so NEW/librnnt_b200.so

Prints same / DIFF / missing per function and exits 1 on any difference or on a function that only one side has."""
import re
import subprocess
import sys


def funcs(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
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


def main():
    old, new = funcs(sys.argv[1]), funcs(sys.argv[2])
    n_same = n_bad = 0
    for name in sorted(set(old) | set(new)):
        if name not in old or name not in new:
            print("missing in %s: %s" % ("OLD" if name not in old else "NEW", name))
            n_bad += 1
            continue
        same = old[name] == new[name]
        n_same += same
        n_bad += not same
        print("%-5s %s (%d instructions)" % ("same" if same else "DIFF", name, len(new[name])))
    print("identical: %d, different or missing: %d" % (n_same, n_bad))
    sys.exit(1 if n_bad or not n_same else 0)


if __name__ == "__main__":
    main()
