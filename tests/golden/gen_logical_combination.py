#!/usr/bin/env python
"""Regenerate tests/golden/logical_combination.json from the reference's
unit/hyperscan/logical_combination.cpp (intel/hyperscan 5.4.2).

Each block-mode test there compiles expressions, flags and ids with
hs_compile_multi, scans one string with hs_scan and lists every callback as
MatchRecord(offset, id), in order.  This keeps exactly that data: the test's name,
the expressions, flags (as the HS_FLAG_* names), ids, the corpus and the expected
(offset, id) sequence.  The streaming test (HS_MODE_STREAM) is left out.

usage: gen_logical_combination.py [path to unit/hyperscan/logical_combination.cpp]
"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/unit/hyperscan/logical_combination.cpp"


def c_strings(text):
    """The concatenated C string literals of `text` (adjacent literals join)."""
    return "".join(m.group(1) for m in re.finditer(r'"((?:[^"\\]|\\.)*)"', text)).encode().decode("unicode_escape")


def braces(body, name):
    m = re.search(r"\b" + name + r"\[\]\s*=\s*\{(.*?)\};", body, re.S)
    return m.group(1)


def main():
    src = open(SRC).read()
    cases = []
    for m in re.finditer(r"TEST\(LogicalCombination,\s*(\w+)\)\s*\{(.*?)\n\}", src, re.S):
        name, body = m.group(1), m.group(2)
        if "HS_MODE_STREAM" in body:
            continue
        data = c_strings(re.search(r"string data\s*=\s*(.*?);", body, re.S).group(1))
        exprs = [c_strings(e) for e in re.findall(r'"(?:[^"\\]|\\.)*"', braces(body, "expr"))]
        flags = [[f for f in re.findall(r"HS_FLAG_\w+", x)] for x in braces(body, "flags").split(",")]
        ids = [int(x) for x in re.findall(r"\d+", braces(body, "ids"))]
        matches = [[int(a), int(b)] for a, b in re.findall(r"MatchRecord\((\d+),\s*(\d+)\)", body)]
        count = int(re.search(r"ASSERT_EQ\((\d+)U, c\.matches\.size\(\)\)", body).group(1))
        assert len(exprs) == len(flags) == len(ids) and count == len(matches), name
        cases.append({"name": name, "expressions": exprs, "flags": flags, "ids": ids, "data": data,
                      "matches": matches})
    out = {"source": "intel/hyperscan 5.4.2 unit/hyperscan/logical_combination.cpp",
           "generator": "tests/golden/gen_logical_combination.py", "cases": cases}
    with open(os.path.join(HERE, "logical_combination.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(len(cases), "cases")


if __name__ == "__main__":
    main()
