"""Compile-time check of the K12 kernel (no GPU needed): every conv_tc_kernel instantiation fits the consumers' register
budget without spilling, and ptxas keeps its wgmmas asynchronous.  If ptxas cannot prove that a pending wgmma's registers
stay untouched, or runs out of registers for them, it serialises every wgmma of the kernel and says so only in its -v
report."""
import os
import re
import shutil
import subprocess

import pytest

from xuance_b200 import build

NVCC = build._nvcc()


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not available")
def test_conv_tc_kernels_no_spills_no_serialised_wgmma(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [NVCC] + flags + ["-c", os.path.join(build.CSRC, "conv_tc.cu"), "-o", str(tmp_path / "conv_tc.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*conv_tc_kernel\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = int(m.group(1)) + int(m.group(2))
            cur = None
    assert len(kernels) >= 40, log                            # 6 plane pairs x tile widths x forward / weight gradient
    assert {k: v for k, v in kernels.items() if v} == {}
    assert not [l for l in log.splitlines() if "serialized" in l], log
