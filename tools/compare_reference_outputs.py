"""Check that a regenerated tests/golden/reference_outputs.npz keeps every record of the previous one.

    python tools/compare_reference_outputs.py OLD.npz NEW.npz

Every key of OLD must be in NEW with the same dtype, shape and bytes; keys only in NEW are listed as added.
"""
import sys

import numpy as np

old, new = (dict(np.load(p)) for p in sys.argv[1:3])
changed = [k for k in old if k not in new or old[k].dtype != new[k].dtype or old[k].shape != new[k].shape
           or old[k].tobytes() != new[k].tobytes()]
added = sorted(k for k in new if k not in old)
print("old keys: %d, new keys: %d, added: %d, old keys missing or changed: %d" % (len(old), len(new), len(added),
                                                                                   len(changed)))
for k in changed:
    print("CHANGED", k)
print("added keys (first 10):", added[:10])
sys.exit(1 if changed else 0)
