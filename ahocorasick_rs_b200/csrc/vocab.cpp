// vocab.cpp -- host-side construction of the vocabulary image (vocab.h): a copy of a Standard dense DFA, the depth of
// every state, one record per id, tail_hit of every id (one pass over the entry bytes) and the bytes themselves.
#include "vocab.h"

#include <cstring>
#include <string>

#include "automaton.h"

namespace acb {
namespace {

inline uint64_t align16(uint64_t x) { return (x + 15) & ~uint64_t(15); }

}  // namespace

std::string vocab_check(const uint64_t *offsets, uint64_t n_vocab) {
    if (n_vocab > kVocabMaxIds) return "n_vocab " + std::to_string(n_vocab) + " exceeds " + std::to_string(kVocabMaxIds) + " ids";
    if (offsets[0] != 0) return "offsets[0] must be 0";
    for (uint64_t t = 0; t < n_vocab; t++)
        if (offsets[t + 1] < offsets[t]) return "offsets decrease at id " + std::to_string(t);
    if (offsets[n_vocab] > kVocabMaxBytes)
        return "the entries hold " + std::to_string(offsets[n_vocab]) + " bytes, more than " + std::to_string(kVocabMaxBytes);
    return std::string();
}

uint64_t vocab_image_bytes(uint64_t dfa_bytes, uint32_t dfa_states, uint64_t n_vocab, uint64_t n_bytes) {
    uint64_t off = align16(sizeof(VocabHeader));
    off = align16(off + dfa_bytes);
    off = align16(off + uint64_t(dfa_states) * 4);
    off = align16(off + n_vocab * sizeof(VocabRec));
    off = align16(off + n_vocab * 4);
    return align16(off + n_bytes);
}

void vocab_image_build(const Automaton &dfa, uint64_t extra, const uint8_t *blob, const uint64_t *offsets, uint64_t n_vocab,
                       uint8_t *out) {
    const ImageHeader &ih = dfa.hdr;
    const uint64_t n_bytes = offsets[n_vocab];
    VocabHeader h{};
    h.magic = kVocabMagic;
    h.n_vocab = (uint32_t)n_vocab;
    h.n_states = ih.n_states;
    h.n_cols = ih.n_cols;
    h.max_pat_len = ih.n_patterns ? ih.max_pat_len : 0;
    h.extra_dfa_bytes = extra;
    uint64_t off = align16(sizeof(VocabHeader));
    h.off_dfa = off;
    off = align16(off + dfa.image.size());
    h.off_depth = off;
    off = align16(off + uint64_t(ih.n_states) * 4);
    h.off_recs = off;
    off = align16(off + n_vocab * sizeof(VocabRec));
    h.off_tail = off;
    off = align16(off + n_vocab * 4);
    h.off_bytes = off;
    h.total_bytes = align16(off + n_bytes);
    h.off_trans = h.off_dfa + ih.off_trans;
    h.off_colmap = h.off_dfa + ih.off_colmap;
    h.off_match_off = h.off_dfa + ih.off_match_off;
    h.off_match_pid = h.off_dfa + ih.off_match_pid;
    std::memset(out, 0, h.total_bytes);
    std::memcpy(out + h.off_dfa, dfa.image.data(), dfa.image.size());

    // depth: a state's trie parent is the target of the one row entry that leads to it from a shallower state; in
    // breadth-first order every state's parent comes first, so one pass over the rows in id order sets them all
    const uint32_t *T = reinterpret_cast<const uint32_t *>(dfa.image.data() + ih.off_trans);
    const uint8_t *colmap = dfa.image.data() + ih.off_colmap;
    uint32_t *depth = reinterpret_cast<uint32_t *>(out + h.off_depth);
    std::vector<uint8_t> seen(ih.n_states, 0);
    seen[kDead] = seen[kRoot] = 1;
    for (uint32_t s = kRoot; s < ih.n_states; s++)
        for (uint32_t c = 0; c < ih.n_cols; c++) {
            const uint32_t t = T[uint64_t(s) * ih.n_cols + c] & kStateMask;
            if (!seen[t] && t > s) {   // a child: failure edges go to shallower (smaller) states, already seen
                seen[t] = 1;
                depth[t] = depth[s] + 1;
            }
        }
    h.lvl2 = ih.n_states;
    for (uint32_t s = kRoot; s < ih.n_states; s++)
        if (depth[s] >= 2) {
            h.lvl2 = s;
            break;
        }

    VocabRec *recs = reinterpret_cast<VocabRec *>(out + h.off_recs);
    int32_t *tail = reinterpret_cast<int32_t *>(out + h.off_tail);
    uint8_t *bytes = out + h.off_bytes;
    if (n_bytes) std::memcpy(bytes, blob, n_bytes);
    uint32_t hits = 0;
    for (uint64_t t = 0; t < n_vocab; t++) {
        const uint32_t a = (uint32_t)offsets[t], len = (uint32_t)(offsets[t + 1] - offsets[t]);
        recs[t] = VocabRec{a, len};
        int32_t last = -1;
        uint32_t s = kRoot;
        for (uint32_t j = 0; j < len; j++) {
            const uint32_t e = T[uint64_t(s) * ih.n_cols + colmap[blob[a + j]]];
            if (e & kMatchFlag) last = (int32_t)j;
            s = e & kStateMask;
        }
        tail[t] = last;
        hits += last >= 0;
    }
    h.n_tail_hits = hits;
    std::memcpy(out, &h, sizeof(h));
}

}  // namespace acb
