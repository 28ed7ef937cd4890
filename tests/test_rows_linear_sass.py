"""What ptxas makes of the independent-row whole-attempt kernel (k_linear_rows_attempt, tdq_attempt.cu), checked without a
GPU: the same properties test_attempt_sass.py keeps for k_linear_attempt.  Its tile chain runs the same serial stage
sequence with per-row coefficients read from a shared-memory row table, so
  - no spills and no stack frame at one CTA of 256 threads per SM (255 registers at most);
  - no generic LD between the first and the last HGMMA: the row table, the pair pointers and the staged error terms are
    read with 32-bit ld.shared, the row buffer and the output times with global loads.
Both instantiations (dopri5, bosh3) are checked.  Needs nvcc and cuobjdump (skipped without them).
"""
import os
import re
import shutil
import subprocess

import pytest

from torchdiffeq_b200.csrc import build

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")
SRC = os.path.join(build.HERE, "tdq_attempt.cu")
KERNELS = {"dopri5": "k_linear_rows_attemptILi6E", "bosh3": "k_linear_rows_attemptILi3E"}

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)),
                                reason="nvcc / cuobjdump not available")

_INSN = re.compile(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_]*)(\S*)")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    out = tmp_path_factory.mktemp("rows_attempt_sass")
    obj = str(out / "tdq_attempt.o")
    cmd = [NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", SRC, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _ptxas_entry(log, key):
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    hits = [b for b in blocks[1:] if key in b.split("\n", 1)[0]]
    assert len(hits) == 1, "expected one ptxas entry for %s" % key
    return hits[0]


def _function(sass, key):
    parts = re.split(r"\n\s*Function : ", sass)
    hits = [p for p in parts[1:] if key in p.split("\n", 1)[0]]
    assert len(hits) == 1, "expected one SASS function for %s" % key
    ops = []
    for line in hits[0].splitlines():
        m = _INSN.match(line)
        if m:
            ops.append(m.group(1) + m.group(2))
    return ops


@pytest.mark.parametrize("tableau", sorted(KERNELS))
def test_rows_attempt_kernel_does_not_spill(compiled, tableau):
    log, _ = compiled
    entry = _ptxas_entry(log, KERNELS[tableau])
    assert re.search(r"\b0 bytes stack frame", entry), entry
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", entry)
    assert m and (int(m.group(1)), int(m.group(2))) == (0, 0), entry
    regs = re.search(r"Used (\d+) registers", entry)
    assert regs and int(regs.group(1)) <= 255, entry


@pytest.mark.parametrize("tableau", sorted(KERNELS))
def test_rows_attempt_kernel_no_generic_load_between_products(compiled, tableau):
    _, sass = compiled
    ops = _function(sass, KERNELS[tableau])
    mma = [i for i, op in enumerate(ops) if op.startswith("HGMMA")]
    assert mma, "no HGMMA in the %s instantiation" % tableau
    generic = [ops[i] for i in range(mma[0], mma[-1]) if ops[i] == "LD" or ops[i].startswith("LD.")]
    assert not generic, "%d generic loads between the first and last HGMMA: %s" % (len(generic), sorted(set(generic)))
