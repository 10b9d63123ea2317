"""Code generation of the 3xTF32 group-MLP kernel (csrc/sa_mlp_tc.cu), checked from the compiler's own report (no GPU):
every instantiation of sa_mlp_tc_kernel keeps its accumulators in registers (no spills to local memory) and ptxas
does not serialise its asynchronous warpgroup MMAs or insert waits of its own.  Either would cost the kernel its
overlap of MMAs, epilogues and gathers without changing a single result, so no numerical test would notice."""
import os
import re
import shutil
import subprocess

import pytest

from toothgroupnetwork_b200 import build

KERNEL = "sa_mlp_tc_kernel"


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    obj = tmp_path_factory.mktemp("sa_tc") / "sa_mlp_tc.o"
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "sa_mlp_tc.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return res.stdout + res.stderr


def _per_kernel(report):
    """{mangled name: [report lines]} for every sa_mlp_tc_kernel entry; the notes ptxas prints before an entry's
    'Compiling entry function' line name the function they belong to."""
    out = {}
    current = None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if KERNEL in m.group(1) else None
            if current:
                out.setdefault(current, [])
            continue
        m = re.search(r"in (?:the )?function '(\w+)", line)
        if m and KERNEL in m.group(1):
            out.setdefault(m.group(1), []).append(line)
        elif current:
            out[current].append(line)
    return out


def test_every_instantiation_is_reported(ptxas_report):
    kernels = _per_kernel(ptxas_report)
    # 4 or 2 tile groups per CTA x inner width 16 / 32 / 48 / 64
    assert len(kernels) == 8, sorted(kernels)


def test_no_spills(ptxas_report):
    for name, lines in _per_kernel(ptxas_report).items():
        spills = [l for l in lines if "spill" in l]
        assert spills, f"{name}: no spill line in the ptxas report"
        for l in spills:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and m.group(1) == "0" and m.group(2) == "0", f"{name}: {l.strip()}"


def test_wgmma_not_serialised(ptxas_report):
    for name, lines in _per_kernel(ptxas_report).items():
        bad = [l.strip() for l in lines
               if re.search(r"\(C75(1[4-8]|20)\)", l) or "mma_async instructions are serialized" in l
               or "warpgroup.wait is injected" in l]
        assert not bad, f"{name}:\n" + "\n".join(bad)
