"""The generic row step of the tick kernel, read from the SASS of the sm_90a build of libgsim.so
(nvcc cross-compiles without a GPU, cuobjdump disassembles without one).

A single-GPU mailbox post is a fire-and-forget global reduction (red.global.gpu.or), not a generic
fetching atomic; the gossip turn keeps its per-broadcast send counts in a register, not in a local array;
and the step stays an out-of-line call, so that the kernel's loops keep 64 registers (4 CTAs per SM)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "consul_b200", "libgsim.so")
KERNEL = "gs_tick_kernelILb0EE"  # the instantiation without network coordinates (the bench pool's)

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not installed")


def _kernel_listing():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    ins, on = [], False
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            on = KERNEL in m.group(1)
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if on and m:
            ins.append((int(m.group(1), 16), m.group(2)))
    assert ins, KERNEL
    return ins


def _calls(body):
    return {int(m.group(1), 16) for s in body for m in [re.search(r"CALL\.REL\.NOINC (0x[0-9a-f]+)", s)] if m}


@pytest.fixture(scope="module")
def row_step():
    """The instructions of the out-of-line unimpaired row step: the listing of a kernel holds the
    functions it calls after its own body, each starting at a call target; the step is the largest
    function the kernel body calls (the impaired instantiation is called from the step)."""
    ins = _kernel_listing()
    starts = sorted(_calls(s for _, s in ins))
    bounds = [0] + starts + [ins[-1][0] + 16]
    funcs = {a: [s for x, s in ins if a <= x < b] for a, b in zip(bounds, bounds[1:])}
    step = max(_calls(funcs[0]), key=lambda a: len(funcs[a]))
    assert len(funcs[step]) > 1000, len(funcs[step])
    return [re.sub(r"^@!?U?P\w+\s+", "", s).split()[0] for s in funcs[step]]


def test_single_gpu_mailbox_posts_are_global_reductions(row_step):
    assert not [op for op in row_step if op.startswith("ATOM.E.OR")]   # no generic fetching atomic OR
    assert row_step.count("REDG.E.OR.STRONG.GPU") >= 1                 # red.global.gpu.or.b32


def test_tick_kernel_keeps_64_registers_and_its_stack_frame():
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    res = re.findall(r"Function \S*(gs_tick_kernelILb[01]EE)\S*:\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert len(res) == 2, out
    stack = {name: int(s) for name, _, s in res}
    assert all(int(r) <= 64 for _, r, _ in res), res
    # 384 B with the gossip turn's send counts in a local array
    assert stack["gs_tick_kernelILb0EE"] < 384, stack
