"""Code generation of both group-MLP kernels of csrc/sa_mlp_tc.cu, checked from the compiler's own report (no GPU): the
split-fp16 sa_mlp_tc_kernel and its 3xTF32 fallback sa_mlp_tc3_kernel, at every instantiation, keep their accumulators in
registers (no spills), fit 128 registers per thread (four tile groups of 128 threads in one 64K-register SM), and ptxas
neither serialises their asynchronous warpgroup MMAs nor inserts waits of its own."""
import re

import pytest

from test_cpu_sa_tc_codegen import ptxas_report  # noqa: F401  (the module-scoped ptxas run)

KERNELS = ("sa_mlp_tc_kernel", "sa_mlp_tc3_kernel")


def _entries(report, kernel):
    """{mangled name: [report lines]} for every entry of `kernel` (by its mangled-name component)"""
    tag = f"{len(kernel)}{kernel}I"
    out, current = {}, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if tag in m.group(1) else None
            if current:
                out.setdefault(current, [])
            continue
        m = re.search(r"in (?:the )?function '(\w+)", line)
        if m:
            if tag in m.group(1):
                out.setdefault(m.group(1), []).append(line)
        elif current:
            out[current].append(line)
    return out


@pytest.mark.parametrize("kernel", KERNELS)
def test_every_instantiation_is_reported(ptxas_report, kernel):  # noqa: F811
    assert len(_entries(ptxas_report, kernel)) == 8          # 4 or 2 tile groups x inner width 16 / 32 / 48 / 64


@pytest.mark.parametrize("kernel", KERNELS)
def test_no_spills_and_four_groups_fit(ptxas_report, kernel):  # noqa: F811
    for name, lines in _entries(ptxas_report, kernel).items():
        spills = [l for l in lines if "spill" in l]
        assert spills, f"{name}: no spill line in the ptxas report"
        for l in spills:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l)
            assert m and m.group(1) == "0" and m.group(2) == "0", f"{name}: {l.strip()}"
        regs = [int(m.group(1)) for l in lines for m in [re.search(r"Used (\d+) registers", l)] if m]
        assert regs and max(regs) <= 128, f"{name}: {regs}"


@pytest.mark.parametrize("kernel", KERNELS)
def test_wgmma_not_serialised(ptxas_report, kernel):  # noqa: F811
    for name, lines in _entries(ptxas_report, kernel).items():
        bad = [l.strip() for l in lines
               if re.search(r"\(C75(1[4-8]|20)\)", l) or "mma_async instructions are serialized" in l
               or "warpgroup.wait is injected" in l]
        assert not bad, f"{name}:\n" + "\n".join(bad)
