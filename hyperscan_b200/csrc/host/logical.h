/*
 * logical.h -- logical combinations of expressions (HS_FLAG_COMBINATION): the
 * parser of the combination grammar and the keys, operation tree and per-combination
 * records a database carries for them (src/parser/logical_combination.cpp,
 * src/util/logical.h:42-72, src/util/report_manager.cpp:98-153).
 *
 * Every expression id that some combination names gets a logical key (lkey), in
 * order of first mention; every combination gets a combination key (ckey), in
 * order of appearance.  The operations of all combinations form one array whose
 * ids follow the lkeys (lkeyCount + index); a combination's operations are the
 * contiguous range start..result of it, evaluated in order (isLogicalCombination,
 * src/report.h:190-245).
 */
#ifndef HSB200_LOGICAL_H
#define HSB200_LOGICAL_H

#include <cstdint>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../ref_layout.h"

/* (included by rose_build.h after CompileError, which the parser throws) */

namespace hsb {

struct LogicalSet {
    std::map<u32, u32> lkeyOf;                /* expression id -> lkey */
    std::map<u32, u32> ckeyOf;                /* combination id -> ckey */
    std::map<u32, std::set<u32>> ckeysOfLkey; /* lkey -> the combinations that name it */
    std::vector<LogicalOp> tree;
    std::vector<CombInfo> combs;              /* by ckey */

    bool empty() const { return combs.empty(); }
    u32 lkey(u32 id) const {
        auto it = lkeyOf.find(id);
        return it == lkeyOf.end() ? INVALID_LKEY : it->second;
    }

    /* Parse one combination expression.  Throws CompileError (index -1: the caller
     * supplies it) with the reference's wording: "Unknown character at index 6.",
     * "Not enough operand at index 11.", "No logical operation.", ... */
    void add(u32 id, const char *text, u32 ekey, u64 minOffset, u64 maxOffset);

    /* After the last add(): give the operations their final ids (after the lkeys). */
    void renumber();
};

namespace logical_detail {

/* operation ids are provisional while parsing: this bit marks an index into the tree */
static const u32 OP_MARK = 0x80000000u;

struct Located {
    std::string what;
};

struct PendingOp {
    u32 op;    /* LogicalOpType: NOT binds tightest, then AND, then OR */
    u32 depth; /* parenthesis depth it was read at */
};

/* Does the operator on top of the stack apply before `next` is pushed?  A deeper operator
 * always does; at one depth, one that binds at least as tightly does (so equal operators
 * group to the left). */
inline bool appliesFirst(const PendingOp &top, const PendingOp &next) {
    if (top.depth != next.depth) {
        return top.depth > next.depth;
    }
    return top.op <= next.op;
}

} // namespace logical_detail

inline void LogicalSet::add(u32 id, const char *text, u32 ekey, u64 minOffset, u64 maxOffset) {
    const u32 ckey = ckeyOf.emplace(id, (u32)ckeyOf.size()).first->second;
    std::vector<logical_detail::PendingOp> ops;
    std::vector<u32> operands; /* lkeys and OP_MARK | tree index */
    u32 start = INVALID_LKEY;
    u32 depth = 0;
    size_t numStart = SIZE_MAX; /* first digit of the id being read */
    size_t i = 0;
    /* the id that ends at i, if one is being read */
    auto endNumber = [&]() {
        if (numStart == SIZE_MAX) {
            return;
        }
        if (i - numStart > 9) {
            throw logical_detail::Located{"Expression id too large"};
        }
        u32 v = 0;
        for (size_t k = numStart; k < i; k++) {
            v = v * 10 + (u32)(text[k] - '0');
        }
        numStart = SIZE_MAX;
        const u32 lk = lkeyOf.emplace(v, (u32)lkeyOf.size()).first->second;
        ckeysOfLkey[lk].insert(ckey);
        operands.push_back(lk);
    };
    auto apply = [&]() {
        if (operands.empty()) {
            throw logical_detail::Located{"Not enough operand"};
        }
        LogicalOp o;
        o.op = ops.back().op;
        o.ro = operands.back();
        operands.pop_back();
        o.lo = 0;
        if (o.op != LOGICAL_OP_NOT) {
            if (operands.empty()) {
                throw logical_detail::Located{"Not enough operand"};
            }
            o.lo = operands.back();
            operands.pop_back();
        }
        o.id = logical_detail::OP_MARK | (u32)tree.size();
        tree.push_back(o);
        operands.push_back(o.id);
        ops.pop_back();
        if (start == INVALID_LKEY) {
            start = o.id;
        }
    };
    try {
        for (; text[i]; i++) {
            const char c = text[i];
            if (c >= '0' && c <= '9') {
                if (numStart == SIZE_MAX) {
                    numStart = i;
                }
                continue;
            }
            endNumber();
            if (c == ' ') {
                continue;
            }
            if (c == '(') {
                depth++;
            } else if (c == ')') {
                if (!depth) {
                    throw logical_detail::Located{"Not enough left parentheses"};
                }
                depth--;
            } else if (c == '!' || c == '&' || c == '|') {
                const logical_detail::PendingOp next{
                    c == '!' ? (u32)LOGICAL_OP_NOT : c == '&' ? (u32)LOGICAL_OP_AND : (u32)LOGICAL_OP_OR, depth};
                while (!ops.empty() && logical_detail::appliesFirst(ops.back(), next)) {
                    apply();
                }
                ops.push_back(next);
            } else {
                throw logical_detail::Located{"Unknown character"};
            }
        }
        if (depth) {
            throw logical_detail::Located{"Not enough right parentheses"};
        }
        endNumber();
        while (!ops.empty()) {
            apply();
        }
        if (operands.size() != 1) {
            throw logical_detail::Located{"Not enough operator"};
        }
    } catch (const logical_detail::Located &e) {
        throw CompileError{e.what + " at index " + std::to_string(i) + ".", -1};
    }
    if (start == INVALID_LKEY) {
        throw CompileError{"No logical operation.", -1};
    }
    CombInfo ci;
    ci.id = id;
    ci.ekey = ekey;
    ci.start = start;
    ci.result = operands.back();
    ci.min_offset = minOffset;
    ci.max_offset = maxOffset;
    combs.push_back(ci);
}

inline void LogicalSet::renumber() {
    const u32 n = (u32)lkeyOf.size();
    auto fix = [n](u32 &k) {
        if (k & logical_detail::OP_MARK) {
            k = (k & ~logical_detail::OP_MARK) + n;
        }
    };
    for (LogicalOp &o : tree) {
        fix(o.id);
        fix(o.lo);
        fix(o.ro);
    }
    for (CombInfo &ci : combs) {
        fix(ci.start);
        fix(ci.result);
    }
}

} // namespace hsb
#endif
