/*
 * pair_table.h -- first-stage tables of the class-pair filter (FK_PAIR32,
 * device/kernels.h): a byte -> 5-bit class map for each of the two bytes of a
 * sample and the 1024-entry table indexed by the class pair.
 *
 * The reference's FDR indexes its table with the low `domain` bits of two input
 * bytes (src/fdr/fdr.c:157-170, table built by setupTab,
 * src/fdr/fdr_compile.cpp:527-632).  On the GPU a lookup is only bank-conflict
 * free if every lane owns a copy of the table, which caps it at 1024 entries;
 * ten raw bits of two bytes make a poor key, so the key is built from byte
 * CLASSES chosen for the literal set: bytes no literal uses collapse into one
 * class, the rest are merged greedily where the modelled candidate rate grows
 * least.  Any such table is a sound (superset) filter; confirm decides.
 */
#ifndef HSB200_PAIR_TABLE_H
#define HSB200_PAIR_TABLE_H

#include <vector>

#include "db_walk.h"

namespace hsb {

struct PairTables {
    u32 classWord[256]; /* c0(b) << 7 | c1(b) << 12: c0 = class as first byte of a sample, c1 = as second */
    u32 pair[1024];     /* [c1 << 5 | c0]: byte i = 8 buckets, bit SET = no literal of the bucket
                         * can end at sample position + i + slotBase */
    u32 nClass0, nClass1;
    double modelRate;   /* modelled candidates per byte on uniformly random printable ASCII */
};

/* tails: LitInfo v/msk/size + bucket of every literal (loadReportRules); slotBase:
 * 0 = suffix slots 0..3 (sets with one-byte literals), 1 = slots 1..4. */
void buildPairTables(const std::vector<LitTail> &tails, u32 slotBase, PairTables *out,
                     u32 maxClass0 = 32, u32 maxClass1 = 32);

} // namespace hsb
#endif
