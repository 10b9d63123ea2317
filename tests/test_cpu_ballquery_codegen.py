"""Code generation of the grid ball query (csrc/ballquery_grid.cu), checked from the compiler's own report (no GPU): the build
and query kernels keep everything in registers and shared memory -- no spills and no local-memory stack frame.  A spill in
the query kernel's per-lane segment search would cost time without changing a single result."""
import os
import re
import shutil
import subprocess

import pytest

from toothgroupnetwork_b200 import build

KERNELS = ("bq_grid_build_kernel", "ball_query_grid_kernel")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    obj = tmp_path_factory.mktemp("bq_grid") / "ballquery_grid.o"
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "ballquery_grid.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return res.stdout + res.stderr


def _per_kernel(report):
    """{mangled name: [report lines]} for the entries of KERNELS."""
    out, current = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            if current:
                out.setdefault(current, [])
            continue
        m = re.search(r"(?:for|in (?:the )?function) '(\w+)'", line)
        if m and any(k in m.group(1) for k in KERNELS):
            out.setdefault(m.group(1), []).append(line)
        elif current:
            out[current].append(line)
    return out


def test_every_kernel_is_reported(ptxas_report):
    names = list(_per_kernel(ptxas_report))
    assert sum("bq_grid_build_kernel" in n for n in names) == 1, names
    assert sum("ball_query_grid_kernel" in n for n in names) == 2, names     # int32 and int64 outputs


def test_no_spills_no_local_memory(ptxas_report):
    for name, lines in _per_kernel(ptxas_report).items():
        text = "\n".join(lines)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert m, f"{name}: no frame / spill line in the ptxas report"
        assert m.groups() == ("0", "0", "0"), f"{name}: {m.group(0)}"
        assert not re.search(r"\d+ bytes lmem", text) or re.search(r"\b0 bytes lmem", text), f"{name}: uses local memory"
