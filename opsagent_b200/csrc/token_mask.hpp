// token_mask.hpp — grammar masks over a TOKEN vocabulary (byte-level BPE of a real checkpoint, or the synthetic byte-level ids).
//
// The ToolPrompt grammar (grammar.hpp) is a byte automaton.  A token is allowed in a state iff walking ALL of its bytes through the
// automaton from that state succeeds (the JSON may complete exactly at the token's last byte, never before it).  Allowed sets are
// computed by a depth-first walk of a byte trie of the vocabulary — a rejected byte prunes every token below it, so literal states
// (one allowed byte) cost microseconds and string states visit only the printable-ASCII part of the trie — and cached per
// (grammar, canonical state).  The bitset [ceil(vocab/32)] goes to the device once per state; the LM-head epilogue of the GEMM
// applies it while it computes the row arg-max (gemm_wgmma.cu EPI_LOGITS), so constrained rows cost no extra kernel.
// This is what lets `json_mode` / OpenAI function calling work on real checkpoints (reference consumer: pkg/assistants/simple.go:366-382
// json.Unmarshal into tools.ToolPrompt, pkg/tools/tool.go:29-38).  oracle/oracle.py restates the rule by brute force for the tests.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "grammar.hpp"

namespace oa {

// tokens longer than this are never allowed under a grammar (long whitespace / punctuation runs): bounds the state canonicalisation below
constexpr int GRAMMAR_MAX_TOKEN_BYTES = 32;

class TokenTrie {
public:
    // id_bytes[id] = raw bytes of token id; empty = not a text token (control tokens, unused ids)
    void build(const std::vector<std::string>& id_bytes, int vocab) {
        vocab_ = vocab;
        nodes_.clear(); nodes_.push_back(Node{});
        for (int id = 0; id < (int)id_bytes.size() && id < vocab; ++id) {
            const std::string& b = id_bytes[id];
            if (b.empty() || (int)b.size() > GRAMMAR_MAX_TOKEN_BYTES) continue;
            int n = 0;
            for (unsigned char ch : b) {
                int child = -1;
                for (auto& e : nodes_[n].edges) if (e.first == ch) { child = e.second; break; }
                if (child < 0) { child = (int)nodes_.size(); nodes_[n].edges.push_back({ch, child}); nodes_.push_back(Node{}); }
                n = child;
            }
            nodes_[n].ids.push_back(id);
        }
    }
    int words() const { return (vocab_ + 31) / 32; }
    // out[words()] = bitset of the token ids allowed from cursor c0 (zeroed here)
    void allowed_tokens(const ToolPromptGrammar& g, const ToolPromptGrammar::Cursor& c0, uint32_t* out) const {
        std::fill(out, out + words(), 0u);
        if (g.done_at(c0)) return;
        struct Frame { int node; ToolPromptGrammar::Cursor c; };
        std::vector<Frame> stack; stack.push_back(Frame{0, c0});
        while (!stack.empty()) {
            const Frame f = stack.back(); stack.pop_back();
            for (auto& e : nodes_[f.node].edges) {
                ToolPromptGrammar::Cursor c = f.c;
                if (!g.step(c, e.first)) continue;
                for (int id : nodes_[e.second].ids) out[id >> 5] |= 1u << (id & 31);
                if (!nodes_[e.second].edges.empty() && !g.done_at(c)) stack.push_back(Frame{e.second, c});
            }
        }
    }
private:
    struct Node { std::vector<std::pair<unsigned char, int>> edges; std::vector<int> ids; };
    std::vector<Node> nodes_; int vocab_ = 0;
};

// Cache key of a grammar state.  Inside a string segment the allowed TOKEN set depends on the offset only through (a) how many more
// string bytes fit (capped at the longest admissible token) and (b) how many are still missing before the closing quote is legal.
inline std::string grammar_mask_key(const ToolPromptGrammar& g, const ToolPromptGrammar::Cursor& c) {
    int lo = 0, hi = 0;
    if (g.string_bounds(c, lo, hi)) {
        const int rem = std::min(hi - c.off, GRAMMAR_MAX_TOKEN_BYTES), deficit = std::max(0, lo - c.off);
        return g.state_key(ToolPromptGrammar::Cursor{c.seg, -1 - (rem * 64 + std::min(deficit, 63)), 0});
    }
    return g.state_key(c);
}

}  // namespace oa
