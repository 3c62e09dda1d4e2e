"""What the library computes, and with which kernels, must not depend on the caller's environment.  The one variable its
CUDA sources may read is LION_TIMELINE, a diagnostic that adds timestamp kernels for lion_ctx_timeline."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lion_b200", "csrc")


def test_cuda_sources_read_no_environment_variable_but_the_timeline():
    sources = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
    assert sources, CSRC
    reads = {}
    for path in sources:
        with open(path) as f:
            for m in re.finditer(r"getenv\s*\(([^)]*)\)", f.read()):
                reads.setdefault(m.group(1).strip(), []).append(os.path.basename(path))
    assert sorted(reads) == ['"LION_TIMELINE"'], reads
