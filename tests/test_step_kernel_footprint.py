"""CPU: instruction and local-memory footprint of the one-warp step kernel as built for gather-trade-build (the
headline configuration: Build + ContinuousDoubleAuction + Gather, 64-register variant).

The kernel's speed on the H100 is set by instruction issue and instruction fetch, not by HBM: code that grows inside
it costs time even on paths that never run, and local-memory (stack) traffic goes to L2 because the L1 carve-out is
almost all shared memory.  These budgets turn such growth into a failing test.  They read the built library with
cuobjdump / nvdisasm; no GPU is needed.

The kernel's section holds its own (hot) body followed by the out-of-line callees it needs (auto-reset, device reset,
metric_0 after a reset, the MT19937 twist, dense-log rows, libdevice slow paths).  The budgets below are for the hot
body, the whole section and the per-thread stack frame.  The frame is almost all the out-of-line device reset's
(`device_reset_env` spills about 370 B); the hot body itself touches only a few stack words, and that count has its own
bound.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from ai_economist_b200.build import build_library

# aie_step_kernel<MINB = 4, EXT = false, CS = CS_GTB (Build | CDA | Gather = 0b111)>
C2_KERNEL = "_ZN3aie15aie_step_kernelILi4ELb0ELi7EEEvNS_6DevCfgENS_7DevBufsEii"
# aie_step_kernel<3, false, CS_GTB_TAX (+ PeriodicBracketTax = 0b1111)>
C3_KERNEL = "_ZN3aie15aie_step_kernelILi3ELb0ELi15EEEvNS_6DevCfgENS_7DevBufsEii"

HOT_INSTR_BUDGET = {C2_KERNEL: 12_000, C3_KERNEL: 14_200}      # instructions of the kernel's own body
HOT_LOCAL_BUDGET = {C2_KERNEL: 100, C3_KERNEL: 115}             # STL + LDL sites in the kernel's own body
HOT_SLOT_BUDGET = {C2_KERNEL: 12, C3_KERNEL: 6}                 # distinct 4-byte stack words the kernel's own body touches
SECTION_BYTES_BUDGET = {C2_KERNEL: 410_000, C3_KERNEL: 445_000}  # SASS text of the whole section (16 B per instruction)
STACK_BUDGET = {C2_KERNEL: 560, C3_KERNEL: 512}                 # bytes per thread (cuobjdump -res-usage STACK)


def _tool(name):
    path = shutil.which(name)
    if path is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
        path = cand if os.path.exists(cand) else None
    if path is None:
        pytest.skip("%s not found" % name)
    return path


@pytest.fixture(scope="module")
def lib():
    return build_library()


@pytest.fixture(scope="module")
def disasm(lib):
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([_tool("cuobjdump"), "-xelf", "all", lib], cwd=tmp, check=True, capture_output=True)
        cubins = [f for f in os.listdir(tmp) if f.endswith(".cubin")]
        out = ""
        for f in cubins:
            out += subprocess.run([_tool("nvdisasm"), "-c", os.path.join(tmp, f)], check=True, capture_output=True,
                                  text=True).stdout
    return out


def section_stats(disasm, kernel):
    """(hot-body instructions, hot-body STL/LDL sites, whole-section instructions, hot-body stack words) of one
    kernel's .text section."""
    lines = disasm.splitlines()
    head = [i for i, l in enumerate(lines) if l.startswith("//--") and (".text." + kernel + " ") in l]
    assert head, "kernel %s not found in the library" % kernel
    hot = local = total = 0
    slots = set()
    in_callee = False
    for l in lines[head[0] + 1:]:
        if l.startswith("//--"):
            break
        if l.startswith("$" + kernel + "$"):
            in_callee = True
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", l)
        if not m:
            continue
        total += 1
        if not in_callee:
            hot += 1
            if m.group(1).split(".")[0] in ("STL", "LDL"):
                local += 1
                a = re.search(r"\[R1(?:\+(0x[0-9a-f]+))?\]", l)
                slots.add(int(a.group(1), 16) // 4 if a and a.group(1) else 0)
    return hot, local, total, len(slots)


@pytest.mark.parametrize("kernel", [C2_KERNEL, C3_KERNEL], ids=["c2_gtb_minb4", "c3_tax_minb3"])
def test_step_kernel_text_within_budget(disasm, kernel):
    hot, local, total, slots = section_stats(disasm, kernel)
    assert hot <= HOT_INSTR_BUDGET[kernel], "hot body grew to %d instructions (budget %d)" % (hot, HOT_INSTR_BUDGET[kernel])
    assert local <= HOT_LOCAL_BUDGET[kernel], "hot body has %d STL/LDL sites (budget %d)" % (local, HOT_LOCAL_BUDGET[kernel])
    assert slots <= HOT_SLOT_BUDGET[kernel], "hot body touches %d stack words (budget %d)" % (slots, HOT_SLOT_BUDGET[kernel])
    assert 16 * total <= SECTION_BYTES_BUDGET[kernel], "section text %d B (budget %d)" % (16 * total, SECTION_BYTES_BUDGET[kernel])


@pytest.mark.parametrize("kernel,regs", [(C2_KERNEL, 64), (C3_KERNEL, 80)], ids=["c2_gtb_minb4", "c3_tax_minb3"])
def test_step_kernel_stack_within_budget(lib, kernel, regs):
    out = subprocess.run([_tool("cuobjdump"), "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    m = re.search(r"Function " + re.escape(kernel) + r":\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert m, "kernel %s not found in cuobjdump -res-usage" % kernel
    assert int(m.group(1)) <= regs, "the %d-register variant uses %s registers" % (regs, m.group(1))
    assert int(m.group(2)) <= STACK_BUDGET[kernel], "stack frame %s B (budget %d)" % (m.group(2), STACK_BUDGET[kernel])


def test_unreachable_step_variants_are_not_built(disasm):
    # the 48-register variant (MINB 5) is never chosen by the launch rule
    assert "aie_step_kernelILi5E" not in disasm
