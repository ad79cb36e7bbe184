"""TEST INFRASTRUCTURE ONLY -- never imported by the product (hyperscan_b200/).

oracle/ holds the CPU side of every parity check:

  ref.py        ctypes binding of oracle/_ref/libhsref_<isa>.so = the UNMODIFIED
                reference runtime (intel/hyperscan 5.4.2, hs_runtime's 47 C files
                compiled where they lie by oracle/ref/Makefile) + ref_driver.c.
                Because our host compiler emits reference-format databases, the
                reference's own hs_scan()/hwlmExec() consume the very same bytes
                the H100 kernels consume.  This is the strongest oracle ("kind":
                "reference" in bench.py's cpu_baseline).
  hs_oracle.c   plain-C restatement of the block-mode literal path (FDR / Teddy
                / noodle first stage, hash confirm, pure-literal rose program,
                dedupe / exhaustion), every function citing the reference
                file:line it follows ("kind": "port").  Pinned against the
                reference's own known-answer tests (tests/test_oracle_kat.py)
                and against oracle/_ref on random inputs.
  brute.py      definition-level oracle for literal sets (SURVEY.md section 8c
                "O2"): independent of any table format, so it also checks the
                host compiler.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this package.
"""
