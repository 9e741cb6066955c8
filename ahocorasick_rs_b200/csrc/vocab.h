// vocab.h -- the vocabulary image: which next token ids would complete a string pattern, given the bytes of every id.
//
// A vocabulary is n_vocab byte strings, vocab[t] the bytes of id t (an entry may be empty).  A row's text T is the
// concatenation of vocab[c] over its history after the last BREAK (an id outside [0, n_vocab)); an empty entry adds
// nothing.  Id t COMPLETES a pattern when some admitted pattern occurs in T || vocab[t] with its end inside vocab[t]:
// a Standard overlapping search of T || vocab[t] has a match ending past len(T).  Such a match is at most
// max_pattern_len bytes long, so only the last max_pattern_len - 1 bytes of T matter, and the state a Standard DFA
// reaches over them decides every candidate (vocab.cuh).
//
// The image holds, 16-byte aligned, offsets in bytes from its start:
//   - a Standard dense DFA image (automaton.h, ImageHeader first): a copy of the automaton's own when its kind is
//     Standard, otherwise one built from its patterns with match kind Standard (Automaton::vocab_dfa);
//   - depth[s], the length of the string state s spells (u32[n_states]; breadth-first numbering makes it
//     non-decreasing, so depth[s] <= 1 exactly when s < lvl2);
//   - one record per id, {byte offset, length} into the entry bytes (u32 x 2);
//   - tail_hit[t], the last byte index j of vocab[t] at which the walk FROM THE ROOT over vocab[t] enters a match
//     state, -1 when it never does (i32[n_vocab]);
//   - the entry bytes, one blob.
//
// Index widths: offsets, lengths and tail_hit are 32-bit, so the format holds at most kVocabMaxIds ids and
// kVocabMaxBytes entry bytes in all (ACB_VOCAB_MAX_IDS / ACB_VOCAB_MAX_BYTES in include/acb200.h).
//
// Shared by the host builder (vocab.cpp) and the kernels.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace acb {

struct Automaton;

constexpr uint32_t kVocabMagic = 0x31564341u;   // "ACV1"
constexpr uint64_t kVocabMaxIds = 0x7fffffffull;
constexpr uint64_t kVocabMaxBytes = 0x7fffffffull;

struct VocabHeader {
    uint32_t magic;
    uint32_t n_vocab;
    uint32_t n_states;       // of the DFA
    uint32_t n_cols;
    uint32_t max_pat_len;    // bytes; 0 without patterns
    uint32_t lvl2;           // the first state of depth 2 (n_states when there is none)
    uint32_t n_tail_hits;    // ids with tail_hit >= 0
    uint32_t pad;
    uint64_t extra_dfa_bytes;  // bytes of the DFA built for the vocabulary (0: a copy of the automaton's own)
    uint64_t off_dfa;        // the DFA image (ImageHeader)
    uint64_t off_trans;      // absolute offsets of the DFA's tables, so the kernels need not read its header
    uint64_t off_colmap;
    uint64_t off_match_off;
    uint64_t off_match_pid;
    uint64_t off_depth;      // u32[n_states]
    uint64_t off_recs;       // VocabRec[n_vocab]
    uint64_t off_tail;       // i32[n_vocab]
    uint64_t off_bytes;      // u8[entry bytes]
    uint64_t total_bytes;
};

struct VocabRec {
    uint32_t off, len;
};

// The checks of a vocabulary's shape (n_vocab and the entry offsets: offsets[0] == 0, non-decreasing, the total within
// the limits); an empty string when it is fine, otherwise why not.  Reads offsets[0 .. n_vocab] only.
std::string vocab_check(const uint64_t *offsets, uint64_t n_vocab);

// The image's size for a DFA image of dfa_bytes and dfa_states states.
uint64_t vocab_image_bytes(uint64_t dfa_bytes, uint32_t dfa_states, uint64_t n_vocab, uint64_t n_bytes);

// Writes the image to out (vocab_image_bytes of it) from the Standard DFA `dfa` (extra = its bytes when it was built
// for the vocabulary, 0 when it is the automaton's own).
void vocab_image_build(const Automaton &dfa, uint64_t extra, const uint8_t *blob, const uint64_t *offsets, uint64_t n_vocab,
                       uint8_t *out);

}  // namespace acb
