"""Extract the known-answer vectors of the reference's own tests into reference_vectors.json.

Run with a checkout of the reference (1ytic/warp-rnnt):

    python tests/golden/make_golden.py REFERENCE_DIR

Source: the reference's pytorch_binding/warp_rnnt/test.py (test_one_to_many :34-62,
test_one_to_empty :64-85, test_forward_single :87-121, test_forward_batch :123-188,
test_forward_single_gather :214-257, test_forward_batch_compact :259-336) and
the reference's tensorflow_binding/warp_rnnt_tf/test.py (test_forward_single_inner_gather :227-252).

Only literal data (logits, labels, lengths, expected costs / gradients) is read, via the AST --
no reference code is executed or copied.  Logits are stored raw; the tests apply log_softmax
exactly as the reference tests do (test.py:42, 68, 98, 147, 225, 283).
"""
import ast
import json
import os
import sys

REF_PT = "pytorch_binding/warp_rnnt/test.py"
REF_TF = "tensorflow_binding/warp_rnnt_tf/test.py"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_vectors.json")

WANTED = {"xs", "ys", "xn", "yn", "expected_cost", "expected_costs", "expected_grads"}


def _literal(node):
    """First literal-evaluable thing inside an assignment's value expression."""
    try:
        return ast.literal_eval(node)
    except Exception:
        pass
    if isinstance(node, ast.Call):
        for a in node.args:
            v = _literal(a)
            if v is not None:
                return v
    return None


def extract(root, path, names):
    tree = ast.parse(open(os.path.join(root, path)).read())
    out = {}
    for cls in [n for n in tree.body if isinstance(n, ast.ClassDef)]:
        for fn in [n for n in cls.body if isinstance(n, ast.FunctionDef)]:
            if fn.name not in names:
                continue
            rec = {"source": f"{path}:{fn.lineno}-{fn.end_lineno}"}
            for node in ast.walk(fn):
                if isinstance(node, ast.Assign) and len(node.targets) == 1 \
                        and isinstance(node.targets[0], ast.Name) and node.targets[0].id in WANTED:
                    name = node.targets[0].id
                    if name in rec:          # keep the first (literal) assignment only
                        continue
                    v = _literal(node.value)
                    if v is not None:
                        rec[name] = v
            out[fn.name] = rec
    return out


def main(root):
    vec = extract(root, REF_PT, {"test_one_to_many", "test_one_to_empty", "test_forward_single",
                           "test_forward_batch", "test_forward_single_gather",
                           "test_forward_batch_compact"})
    tf = extract(root, REF_TF, {"test_forward_single_inner_gather"})
    vec.update(tf)
    for k, r in vec.items():
        missing = {"xs", "ys", "xn", "yn", "expected_grads"} - set(r)
        assert not missing, (k, missing)
        assert "expected_cost" in r or "expected_costs" in r, k
    with open(OUT, "w") as f:
        json.dump(vec, f, indent=1)
    print("wrote", OUT, "with", sorted(vec))


if __name__ == "__main__":
    main(sys.argv[1])
