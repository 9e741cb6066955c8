// completions.h -- the "completions" image: which next token ids complete a pattern after a given history.
//
// Id t COMPLETES pattern p after history C when p is a suffix of C || [t], i.e. p[:-1] is a suffix of C and
// p[-1] == t.  So only the suffixes of C that are some p[:-1] matter, and none longer than K - 1 ids (K = the longest
// pattern in tokens).  The image is a reverse trie over the strings p[:-1], at token granularity:
//
//   - the node at depth d stands for a d-token string s; the root is the empty string;
//   - a node's children prepend one more token (s' = [u] || s), contiguous and sorted by u; the token a node prepends
//     lives in a separate u32 array (kid_tok), so the search for a child reads tokens only;
//   - a node's entries are (p[-1], pid) for the patterns with p[:-1] == s, sorted by (token, pid): the root's are the
//     one-token patterns.
//
// The kernel (completions.cuh) walks from the root backwards over the history's last ids; every node on that path is
// a suffix of C that is some p[:-1], and every such suffix is on it, so the entries along the path are exactly the
// completing (token, pid) pairs -- no failure links.  `elink` names the nearest proper ancestor with entries: the
// count and emit modes walk it to report each token once per history.
//
// Shared by the host builder (completions.cpp) and the kernel.
#pragma once
#include <cstdint>
#include <vector>

namespace acb {

constexpr uint32_t kComplMagic = 0x31434341u;   // "ACC1"
constexpr uint32_t kComplNone = 0xffffffffu;

// All offsets are bytes from the start of the image, 16-byte aligned.
struct ComplHeader {
    uint32_t magic;
    uint32_t n_nodes;      // >= 1 (the root)
    uint32_t n_entries;    // = the number of patterns
    uint32_t depth;        // K - 1: the deepest node (0 without patterns)
    uint32_t max_last;     // the largest id that ends a pattern (0 without patterns)
    uint32_t pad[3];
    uint64_t off_nodes;    // ComplNode[n_nodes], breadth-first: the root is node 0
    uint64_t off_kid_tok;  // u32[n_nodes]: the token node v prepends to its parent's string (0 for the root)
    uint64_t off_entries;  // ComplEntry[n_entries]
    uint64_t total_bytes;
};

struct ComplNode {
    uint32_t first_kid, n_kids;        // children: nodes [first_kid, first_kid + n_kids), sorted by kid_tok
    uint32_t first_entry, n_entries;   // entries [first_entry, first_entry + n_entries), sorted by (token, pid)
    uint32_t elink;                    // nearest proper ancestor with entries, kComplNone = none
    uint32_t pad[3];
};

struct ComplEntry {
    uint32_t token;   // p[-1]
    uint32_t pid;
};

// Builds the image from the patterns' token ids: pattern i is ids[offsets[i] .. offsets[i + 1]), non-empty.
// Throws std::runtime_error on an empty pattern or a trie too large for 32-bit indexes.
uint64_t completions_image_build(const uint32_t *ids, const uint64_t *offsets, uint64_t n, std::vector<uint8_t> &out);

}  // namespace acb
