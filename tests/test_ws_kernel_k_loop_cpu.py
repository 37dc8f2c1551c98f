"""CPU test of what ptxas made of the TMA-fed f64 GEMM (csrc/gemm_f64_ws.cuh): in every plain (non-spicy) variant of
`gemm_f64_ws_kernel` in the built library, the k-step loop (the innermost loop that holds the 32 DMMA of a stage) keeps to
the barrier wait, the 48 fragment loads, the DMMAs and the stage release. The lane's fragment offsets stay in registers
and the stage index and phase advance in uniform registers, so the loop holds almost no per-thread integer arithmetic
and no local-memory access. Without that, ptxas rebuilds the swizzled offsets from the thread index in every k-step (60
to 110 LOP3 / IMAD / IADD3 / SHF / LEA per stage), or reloads them from local memory when the epilogue crowds them out,
and the first DMMA of a stage waits for that chain. Skipped when the library has not been built or cuobjdump is not
installed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "faer-rs_b200", "libfaer_b200.so")
INT_ALU = ("LOP3", "IMAD", "IADD3", "SHF", "LEA")


def cuobjdump():
    for path in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if path and os.access(path, os.X_OK):
            return path
    return None


def k_loop(body):
    """instructions of the shortest backward-branch loop holding >= 32 DMMA"""
    ins = [(int(a, 16), op) for a, op in re.findall(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", body)]
    index = {a: i for i, (a, _) in enumerate(ins)}
    best = None
    for i, (a, op) in enumerate(ins):
        m = re.search(r"\bBRA\b.*?0x([0-9a-f]+)", op)
        if m and int(m.group(1), 16) < a and int(m.group(1), 16) in index:
            loop = [o for _, o in ins[index[int(m.group(1), 16)]:i + 1]]
            if sum("DMMA" in o for o in loop) >= 32 and (best is None or len(loop) < len(best)):
                best = loop
    return best


def test_ws_kernel_k_loop_keeps_to_loads_and_dmma():
    tool = cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built libfaer_b200.so and cuobjdump")
    out = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    seen = 0
    for func in re.split(r"\n\s*Function : ", out.stdout)[1:]:
        name = func.split("\n", 1)[0].strip()
        m = re.search(r"gemm_f64_ws_kernelI(Lb[01]E){3}Lb0E", name)
        if not m:
            continue
        seen += 1
        loop = k_loop(func)
        assert loop is not None, name
        ops = [re.sub(r"^@!?U?P\w+\s+", "", o).split()[0].split(".")[0] for o in loop]
        assert ops.count("DMMA") == 32 and ops.count("LDS") == 48, (name, ops.count("DMMA"), ops.count("LDS"))
        alu = sum(ops.count(k) for k in INT_ALU)
        assert alu <= 4, (name, {k: ops.count(k) for k in INT_ALU})
        assert ops.count("STL") == 0 and ops.count("LDL") == 0, (name, ops.count("STL"), ops.count("LDL"))
    # narrow and wide, each for the four operand layouts
    assert seen == 8
