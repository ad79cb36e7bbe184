/*
 * hwlm_build.h -- host-side literal-matcher table builder (interface).
 *
 * Emits HWLM tables (noodle / Teddy / FDR + hash confirm + flood control) in
 * the reference's byte layouts, so the same bytes can be consumed by the H100
 * kernels and by the unmodified reference runtime (used as the parity oracle).
 * Mirrors the role of hwlmBuildProto()/hwlmBuild() (reference:
 * src/hwlm/hwlm_build.cpp:107-212).
 */
#ifndef HSB200_HWLM_BUILD_H
#define HSB200_HWLM_BUILD_H

#include <string>
#include <vector>

#include "../ref_layout.h"

namespace hsb {

/** One literal as the literal matcher sees it: at most 8 bytes (the suffix of
 * the pattern literal; reference: HWLM_LITERAL_MAX_LEN, src/hwlm/hwlm.h:75).
 * For nocase literals `s` holds upper-cased ASCII letters. */
struct HwlmLit {
    std::string s;
    bool nocase = false;
    bool noruns = false;
    u32 id = 0;       /* delivered to the callback; rose: program offset */
    u64 groups = 1;
};

struct HwlmBuildOpts {
    bool allowNoodle = true;
    bool allowTeddy = true;
    bool allowFatTeddy = false; /* 16-bucket Teddy needs an AVX2 reference target */
    int forceEngine = -1;       /* -1 auto; 0 FDR; 3..18 Teddy id (tests) */
    int forceDomain = 0;        /* FDR: 9..15, 0 = auto */
    int forceStride = 0;        /* FDR: 1,2,4, 0 = auto */
    int maxDomain = 15;         /* cap for the auto choice (H100: smem-resident table) */
    bool allowFlood = true;
};

struct HwlmBuildInfo {
    u32 type = 0;     /* HWLM_ENGINE_* */
    u32 engineID = 0;
    u32 domain = 0;
    u32 stride = 0;
    u32 numBuckets = 0;
    u32 numMasks = 0;
};

/** Build a complete HWLM blob (header + engine).  Throws std::runtime_error
 * on resource-limit style failures. */
std::vector<u8> buildHwlm(std::vector<HwlmLit> lits, const HwlmBuildOpts &opts,
                          HwlmBuildInfo *info);

static inline bool isAsciiAlpha(u8 c) {
    return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z');
}
static inline u8 asciiUpper(u8 c) { return (c >= 'a' && c <= 'z') ? c - 0x20 : c; }
static inline u8 asciiLower(u8 c) { return (c >= 'A' && c <= 'Z') ? c + 0x20 : c; }

u32 crc32c(u32 crc, const void *buf, size_t len);

} // namespace hsb
#endif
