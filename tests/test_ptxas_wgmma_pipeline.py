"""Static check on the ptxas reports of the built library (no GPU needed).

ptxas serialises the wgmma instructions of a kernel that contains a function call (a device printf is a call to vprintf):
every MMA then waits for the previous one to retire and the tensor cores idle between them.  It says so with warning
C7510 in the `-Xptxas -v` report that the Makefile keeps in paella_b200/csrc/build/<source>.ptxas.log.
"""
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGS = sorted(glob.glob(os.path.join(ROOT, "paella_b200", "csrc", "build", "*.ptxas.log")))


@pytest.mark.skipif(not LOGS, reason="the library has not been built here")
def test_no_wgmma_kernel_is_serialised_by_ptxas():
    serialised = []
    for path in LOGS:
        with open(path) as f:
            for line in f:
                if "C7510" in line:
                    m = re.search(r"function '([^']+)'", line)
                    serialised.append((os.path.basename(path), m.group(1) if m else line.strip()))
    assert not serialised, serialised
