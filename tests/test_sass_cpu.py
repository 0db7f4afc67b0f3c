"""CPU test: the kernels of mtadgat_pot, of the streaming SPOT push and grow, and of scale.cu compile to the SASS
recorded in tests/golden/spot_sass.json (sha256 of each kernel's `cuobjdump -sass` listing, with the hash of the
anonymous namespace taken out of symbol names).  The SPOT initialisation shares select.cuh, compact.cuh and gpd_fit.cuh
with these kernels; the record shows that it changed none of them.  Skipped under another nvcc release, whose SASS
differs anyway."""
import hashlib
import json
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "spot_sass.json")
# object -> substrings of the pinned kernels' names (None: every kernel in it)
PINNED = {"pot": None, "scale": None, "spot_stream": ["spot_push_kernel", "spot_push_batched_kernel", "spot_grow_kernel"]}


def kernel_digests(cuobjdump, obj):
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_\d+_\w+?_cu_[0-9a-f]{8}", "_GLOBAL__N_", out)
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name:
            funcs[name].append(line)
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in funcs.items()}


def test_shared_spot_kernels_keep_their_sass():
    import __graft_entry__ as ge
    ge.build()
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    golden = json.load(open(GOLDEN))
    release = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout
    if golden["nvcc"] not in release:
        pytest.skip(f"SASS recorded with nvcc {golden['nvcc']}")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    for obj, want in golden["kernels"].items():
        got = kernel_digests(cuobjdump, os.path.join(ge.OBJDIR, obj + ".o"))
        for name, digest in want.items():
            assert got.get(name) == digest, (obj, name)
