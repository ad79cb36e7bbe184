"""hyperscan_b200 -- Python harness around libhs_b200.so, the H100-native
block-mode scan runtime for Hyperscan databases.  The product is the C-ABI
shared library (include/hs_b200.h); see DESIGN.md."""
