// completions.cpp -- host-side construction of the completions image (completions.h): the reverse trie over every
// pattern's p[:-1], numbered breadth-first with each node's children contiguous and sorted by token.
#include "completions.h"

#include <algorithm>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

namespace acb {
namespace {

inline uint64_t align16(uint64_t x) { return (x + 15) & ~uint64_t(15); }

struct CNode {
    std::map<uint32_t, uint32_t> kids;              // prepended token -> node (ordered: the children come out sorted)
    std::vector<std::pair<uint32_t, uint32_t>> own;  // (last token, pid)
};

}  // namespace

uint64_t completions_image_build(const uint32_t *ids, const uint64_t *offsets, uint64_t n, std::vector<uint8_t> &out) {
    std::vector<CNode> nodes(1);
    uint32_t depth = 0, max_last = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t a = offsets[i], len = offsets[i + 1] - offsets[i];
        if (len == 0) throw std::runtime_error("empty pattern at index " + std::to_string(i));
        if (len - 1 > 0x7fffffffull) throw std::runtime_error("pattern too long");
        // p[:-1] from its last token backwards: the node of the last d tokens before p[-1] is at depth d
        uint32_t v = 0;
        for (uint64_t j = a + len - 1; j-- > a;) {
            auto it = nodes[v].kids.find(ids[j]);
            uint32_t c;
            if (it == nodes[v].kids.end()) {
                if (nodes.size() >= 0x7fffffffull) throw std::runtime_error("too many trie nodes");
                c = (uint32_t)nodes.size();
                nodes[v].kids.emplace(ids[j], c);
                nodes.emplace_back();
            } else {
                c = it->second;
            }
            v = c;
        }
        nodes[v].own.emplace_back(ids[a + len - 1], (uint32_t)i);
        depth = std::max<uint32_t>(depth, (uint32_t)(len - 1));
        max_last = std::max(max_last, ids[a + len - 1]);
    }
    if (n > 0x7fffffffull) throw std::runtime_error("too many patterns");
    const uint32_t n_nodes = (uint32_t)nodes.size();

    // breadth-first numbering: node 0 is the root, every node's children are contiguous and sorted by token
    std::vector<uint32_t> order{0};   // new id -> old id
    std::vector<ComplNode> cn(n_nodes);
    std::vector<uint32_t> kid_tok(n_nodes, 0), parent(n_nodes, kComplNone);
    order.reserve(n_nodes);
    for (size_t q = 0; q < order.size(); q++) {
        const CNode &t = nodes[order[q]];
        cn[q].first_kid = (uint32_t)order.size();
        cn[q].n_kids = (uint32_t)t.kids.size();
        for (const auto &kv : t.kids) {
            kid_tok[order.size()] = kv.first;
            parent[order.size()] = (uint32_t)q;
            order.push_back(kv.second);
        }
    }
    std::vector<ComplEntry> entries;
    entries.reserve(n);
    for (uint32_t v = 0; v < n_nodes; v++) {
        std::vector<std::pair<uint32_t, uint32_t>> own = nodes[order[v]].own;
        std::sort(own.begin(), own.end());
        cn[v].first_entry = (uint32_t)entries.size();
        cn[v].n_entries = (uint32_t)own.size();
        for (const auto &e : own) entries.push_back(ComplEntry{e.first, e.second});
        // parents come first in breadth-first order, so their links are set
        const uint32_t p = parent[v];
        cn[v].elink = p == kComplNone ? kComplNone : (cn[p].n_entries ? p : cn[p].elink);
    }

    ComplHeader h{};
    h.magic = kComplMagic;
    h.n_nodes = n_nodes;
    h.n_entries = (uint32_t)entries.size();
    h.depth = depth;
    h.max_last = max_last;
    uint64_t off = align16(sizeof(ComplHeader));
    h.off_nodes = off;
    off = align16(off + uint64_t(n_nodes) * sizeof(ComplNode));
    h.off_kid_tok = off;
    off = align16(off + uint64_t(n_nodes) * 4);
    h.off_entries = off;
    off = align16(off + entries.size() * sizeof(ComplEntry));
    h.total_bytes = off;
    out.assign(off, 0);
    uint8_t *img = out.data();
    std::memcpy(img, &h, sizeof(h));
    std::memcpy(img + h.off_nodes, cn.data(), uint64_t(n_nodes) * sizeof(ComplNode));
    std::memcpy(img + h.off_kid_tok, kid_tok.data(), uint64_t(n_nodes) * 4);
    if (!entries.empty()) std::memcpy(img + h.off_entries, entries.data(), entries.size() * sizeof(ComplEntry));
    return off;
}

}  // namespace acb
