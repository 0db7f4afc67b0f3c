"""Compare two `bench.py --dump-outputs` directories array by array: every .npy must exist in both and be bitwise
equal (NaNs compare by bit pattern).  Exit status 1 on any difference.
usage: compare_dumps.py DIR_A DIR_B"""
import os
import sys

import numpy as np

a_dir, b_dir = sys.argv[1], sys.argv[2]
names = sorted(set(os.listdir(a_dir)) | set(os.listdir(b_dir)))
bad = 0
for name in names:
    pa, pb = os.path.join(a_dir, name), os.path.join(b_dir, name)
    if not (os.path.exists(pa) and os.path.exists(pb)):
        print(f"missing in {'second' if os.path.exists(pa) else 'first'}: {name}")
        bad += 1
        continue
    a, b = np.load(pa), np.load(pb)
    if a.shape != b.shape or a.dtype != b.dtype or not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
        diff = int(np.count_nonzero(a != b)) if a.shape == b.shape else -1
        print(f"differs: {name} shape {a.shape} vs {b.shape}, {diff} elements")
        bad += 1
print(f"{len(names)} arrays, {bad} differ")
sys.exit(1 if bad else 0)
