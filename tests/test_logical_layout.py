"""The bytecode structures of logical combinations, as hyperscan_b200/csrc/ref_layout.h restates them, have
the reference's sizes, offsets and opcode values (src/rose/rose_program.h:189-209 and :701-723,
src/util/logical.h:53-70; measured on the reference's own headers with gcc on x86-64)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (C++ expression on ref_layout.h, the reference's value)
REFERENCE = [
    ("OP_SET_LOGICAL", 62), ("OP_SET_COMBINATION", 63), ("OP_FLUSH_COMBINATION", 64), ("OP_SET_EXHAUST", 65),
    ("OP_LAST_FLUSH_COMBINATION", 66),
    ("sizeof(InstrSetLogical)", 12), ("offsetof(InstrSetLogical, lkey)", 4),
    ("offsetof(InstrSetLogical, offset_adjust)", 8),
    ("sizeof(InstrSetCombination)", 8), ("offsetof(InstrSetCombination, ckey)", 4),
    ("sizeof(InstrFlushCombination)", 1), ("sizeof(InstrLastFlushCombination)", 1),
    ("sizeof(LogicalOp)", 16), ("offsetof(LogicalOp, op)", 4), ("offsetof(LogicalOp, lo)", 8),
    ("offsetof(LogicalOp, ro)", 12),
    ("sizeof(CombInfo)", 32), ("offsetof(CombInfo, ekey)", 4), ("offsetof(CombInfo, start)", 8),
    ("offsetof(CombInfo, result)", 12), ("offsetof(CombInfo, min_offset)", 16),
    ("offsetof(CombInfo, max_offset)", 24),
    ("LOGICAL_OP_NOT", 0), ("LOGICAL_OP_AND", 1), ("LOGICAL_OP_OR", 2),
]


def test_logical_combination_layouts(tmp_path):
    src = tmp_path / "logical_layout.cpp"
    lines = ['#include <cstddef>', '#include "%s"' % os.path.join(ROOT, "hyperscan_b200", "csrc", "ref_layout.h"),
             "using namespace hsb;"]
    lines += ['static_assert((%s) == %d, "%s");' % (e, v, e) for e, v in REFERENCE]
    src.write_text("\n".join(lines) + "\n")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], capture_output=True, text=True)
    if r.returncode and "static assertion" not in r.stderr:
        pytest.fail(r.stderr)
    assert r.returncode == 0, r.stderr
