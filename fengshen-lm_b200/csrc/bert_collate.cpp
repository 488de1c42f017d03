// Host-side MegatronBERT sample assembly: the per-document work of `ErLangShenCollator`
// (fengshen/examples/pretrain_erlangshen_bert/pretrain_erlangshen.py:57-123 and the fengshen/data/data_utils helpers it calls:
// sop_utils.py:2-32, truncate_utils.py:2-19, token_type_utils.py:1-25, mask_utils.py:19-285 with its defaults) in one C call over a
// batch of ALREADY TOKENISED documents. At a GPU training step's rates the Python collator (~50 k tokens/s per core, DESIGN §6) is the
// first thing to starve the step; this leaves tokenisation as the only Python-side cost.
//
// The batch is bit-identical to the Python path, including the state the numpy RandomState is left in: the generator is numpy's
// legacy MT19937 stream (state passed in and out as `RandomState.get_state()` holds it), consumed through numpy's own derived
// draws — random_sample (two 32-bit words -> 53-bit double), randint / shuffle (masked rejection on 32-bit words), and
// choice(p=...) (one random_sample against the normalised cumulative weights, which the caller computes with numpy and passes in).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/fsb200.h"
#include "host_common.h"

namespace {

struct NumpyMT {   // numpy/random/src/mt19937/mt19937.c: key[624] + pos, regenerated when exhausted
  uint32_t* key;
  int32_t pos;
  void refill() {
    constexpr int N = 624, M = 397;
    constexpr uint32_t UPPER = 0x80000000u, LOWER = 0x7fffffffu, MAGIC = 0x9908b0dfu;
    int i = 0;
    for (; i < N - M; ++i) {
      uint32_t y = (key[i] & UPPER) | (key[i + 1] & LOWER);
      key[i] = key[i + M] ^ (y >> 1) ^ ((y & 1u) ? MAGIC : 0u);
    }
    for (; i < N - 1; ++i) {
      uint32_t y = (key[i] & UPPER) | (key[i + 1] & LOWER);
      key[i] = key[i + (M - N)] ^ (y >> 1) ^ ((y & 1u) ? MAGIC : 0u);
    }
    uint32_t y = (key[N - 1] & UPPER) | (key[0] & LOWER);
    key[N - 1] = key[M - 1] ^ (y >> 1) ^ ((y & 1u) ? MAGIC : 0u);
    pos = 0;
  }
  uint32_t next32() {
    if (pos == 624) refill();
    uint32_t y = key[pos++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
  double random_sample() {   // legacy "genrand_res53"
    const uint32_t a = next32() >> 5, b = next32() >> 6;
    return (a * 67108864.0 + b) / 9007199254740992.0;
  }
  // uniform integer in [0, max], max < 2^32: smallest all-ones mask covering max, redraw until it fits
  // (legacy random_interval used by shuffle, and the masked path of randint for int64 with a 32-bit range)
  uint32_t bounded(uint32_t max) {
    if (max == 0) return 0;
    uint32_t mask = max;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    uint32_t v;
    do { v = next32() & mask; } while (v > max);
    return v;
  }
  int64_t randint(int64_t low, int64_t high) { return low + bounded(static_cast<uint32_t>(high - 1 - low)); }
  template <typename T>
  void shuffle(std::vector<T>& v) {   // RandomState.shuffle on a Python list: i = n-1 .. 1, swap with bounded(i)
    for (int64_t i = static_cast<int64_t>(v.size()) - 1; i >= 1; --i) std::swap(v[i], v[bounded(static_cast<uint32_t>(i))]);
  }
};

struct Params {
  const uint8_t* continuation;   // [vocab_table_len]: 1 where the piece starts with "##"
  int64_t vocab_table_len;
  const int32_t* vocab_ids;      // the list random replacements are drawn from (the collator's vocab_id_list order)
  int64_t n_vocab_ids;
  int32_t cls, sep, mask, pad;
  int32_t max_seq_length;
  double prob;
  const double* ngram_cdf;       // normalised cumulative weights of n-gram sizes 1..max_ngrams (numpy-computed)
  int32_t max_ngrams;
};

// mask_utils.py:19-285 with do_whole_word_mask, masking_style='bert', no segmenter, no permutation. `tok` is edited in place;
// positions / labels come back sorted by position.
void mask_tokens(std::vector<int32_t>& tok, const Params& P, NumpyMT& rng, std::vector<int32_t>& positions,
                 std::vector<int32_t>& labels) {
  const int n = static_cast<int>(tok.size());
  std::vector<int32_t> span_start;   // word w covers [span_start[w], span_start[w + 1])
  std::vector<int32_t> members;      // token positions of all words, concatenated (specials are not members)
  for (int i = 0; i < n; ++i) {
    const int32_t t = tok[i];
    if (t == P.cls || t == P.sep) continue;
    const bool cont = t >= 0 && t < P.vocab_table_len && P.continuation[t];
    if (!(cont && !span_start.empty())) span_start.push_back(static_cast<int32_t>(members.size()));
    members.push_back(i);
  }
  span_start.push_back(static_cast<int32_t>(members.size()));
  const int n_words = static_cast<int>(span_start.size()) - 1;
  positions.clear();
  labels.clear();
  if (P.prob == 0) return;
  const double cap = P.prob * n;   // max_predictions_per_seq as the collator passes it (a float)
  const double rounded = std::nearbyint(n * P.prob);   // Python's round(): half to even, the default FP rounding mode
  const double budget = std::fmin(cap, std::fmax(1.0, rounded));
  std::vector<int32_t> order(n_words);
  for (int w = 0; w < n_words; ++w) order[w] = w;
  rng.shuffle(order);
  std::vector<uint8_t> covered(n, 0);
  std::vector<int32_t> original(tok);
  struct Pick { int32_t pos, label; };
  std::vector<Pick> picks;
  auto window_len = [&](int w, int k) {   // tokens in the n-gram of k words starting at word w (clipped at the end)
    const int last = std::min(w + k, n_words);
    return span_start[last] - span_start[w];
  };
  for (int oi = 0; oi < n_words; ++oi) {
    if (static_cast<double>(picks.size()) >= budget) break;
    const int w = order[oi];
    const double u = rng.random_sample();   // np_rng.choice(sizes, p): searchsorted(cdf, u, side='right')
    int k = 0;
    while (k < P.max_ngrams - 1 && u >= P.ngram_cdf[k]) ++k;
    k += 1;
    int len = window_len(w, k);
    while (static_cast<double>(picks.size()) + len > budget && k > 1) len = window_len(w, --k);
    if (static_cast<double>(picks.size()) + len > budget) continue;
    const int32_t* m = members.data() + span_start[w];
    bool clash = false;
    for (int j = 0; j < len; ++j) clash = clash || covered[m[j]];
    if (clash) continue;
    for (int j = 0; j < len; ++j) {
      const int p = m[j];
      covered[p] = 1;
      int32_t put;
      if (rng.random_sample() < 0.8) put = P.mask;
      else if (rng.random_sample() < 0.5) put = original[p];
      else put = P.vocab_ids[rng.randint(0, P.n_vocab_ids)];
      tok[p] = put;
      picks.push_back({p, original[p]});
    }
  }
  rng.shuffle(order);   // the reference shuffles again before its (disabled) permutation pass
  // counting sort by position (positions are unique)
  std::vector<int32_t> label_at(n, -1);
  for (const Pick& pk : picks) label_at[pk.pos] = pk.label;
  for (int i = 0; i < n; ++i)
    if (covered[i]) { positions.push_back(i); labels.push_back(label_at[i]); }
}

}  // namespace

extern "C" int64_t fsb_bert_collate(const int32_t* tokens, const int64_t* sent_offsets, const int64_t* doc_offsets, int64_t n_docs,
                                    const uint8_t* continuation, int64_t vocab_table_len, const int32_t* vocab_ids,
                                    int64_t n_vocab_ids, int32_t cls_id, int32_t sep_id, int32_t mask_id, int32_t pad_id,
                                    int32_t max_seq_length, double masked_lm_prob, const double* ngram_cdf, int32_t max_ngrams,
                                    uint32_t* mt_key, int32_t* mt_pos, int64_t* input_ids, int64_t* attention_mask,
                                    int64_t* token_type_ids, int64_t* labels, int64_t* next_sentence_label) {
  if (!(tokens && sent_offsets && doc_offsets && continuation && vocab_ids && ngram_cdf && mt_key && mt_pos && input_ids &&
        attention_mask && token_type_ids && labels && next_sentence_label) || n_docs < 0 || n_vocab_ids <= 0 ||
      max_seq_length < 4 || max_ngrams < 1 || masked_lm_prob < 0 || masked_lm_prob > 1 || *mt_pos < 0 || *mt_pos > 624) {
    fsb::set_error("bert_collate: null pointer or bad argument (max_seq_length >= 4, 0 <= masked_lm_prob <= 1, max_ngrams >= 1, "
                   "0 <= mt_pos <= 624)");
    return -1;
  }
  NumpyMT rng{mt_key, *mt_pos};
  const Params P{continuation, vocab_table_len, vocab_ids, n_vocab_ids, cls_id, sep_id, mask_id, pad_id, max_seq_length,
                 masked_lm_prob, ngram_cdf, max_ngrams};
  const int64_t L = max_seq_length;
  int64_t row = 0;
  std::vector<int32_t> tok, positions, lab;
  for (int64_t d = 0; d < n_docs; ++d) {
    const int64_t s0 = doc_offsets[d], s1 = doc_offsets[d + 1];
    const int64_t n_sent = s1 - s0;
    if (n_sent <= 0) continue;   // "find empty sentence": the document yields no row
    // segments A / B as [begin, end) ranges of the flat token array (sop_utils.py): sentences [s0, cut) and [cut, s1)
    int64_t cut = s0 + 1;
    bool swapped = false;
    int64_t a0, a1, b0, b1;
    if (n_sent > 1) {
      if (n_sent >= 3) cut = s0 + rng.randint(1, n_sent);
      swapped = rng.random_sample() < 0.5;
      a0 = sent_offsets[s0]; a1 = sent_offsets[cut]; b0 = sent_offsets[cut]; b1 = sent_offsets[s1];
      if (swapped) { std::swap(a0, b0); std::swap(a1, b1); }
    } else {
      a0 = sent_offsets[s0]; a1 = sent_offsets[s1]; b0 = b1 = a1;
    }
    if (a1 - a0 <= 0) continue;   // empty first segment: skipped, AFTER its draws (as the Python path)
    // truncate_utils.py: shorten the longer segment (ties: B) one token at a time, front or back by a coin flip
    while ((a1 - a0) + (b1 - b0) > L - 3) {
      const bool from_a = (a1 - a0) > (b1 - b0);
      const bool front = rng.random_sample() < 0.5;
      if (from_a) { if (front) ++a0; else --a1; } else { if (front) ++b0; else --b1; }
    }
    tok.clear();
    tok.push_back(cls_id);
    tok.insert(tok.end(), tokens + a0, tokens + a1);
    tok.push_back(sep_id);
    const int64_t n_type0 = static_cast<int64_t>(tok.size());
    if (b1 > b0) {
      tok.insert(tok.end(), tokens + b0, tokens + b1);
      tok.push_back(sep_id);
    }
    mask_tokens(tok, P, rng, positions, lab);
    const int64_t n = static_cast<int64_t>(tok.size());
    int64_t* ids = input_ids + row * L;
    int64_t* am = attention_mask + row * L;
    int64_t* tt = token_type_ids + row * L;
    int64_t* lb = labels + row * L;
    for (int64_t i = 0; i < L; ++i) {
      const bool real = i < n;
      ids[i] = real ? tok[i] : pad_id;
      am[i] = real ? 1 : 0;
      tt[i] = real ? (i < n_type0 ? 0 : 1) : pad_id;   // the reference pads token types with the PAD id as well
      lb[i] = -100;
    }
    for (size_t j = 0; j < positions.size(); ++j) lb[positions[j]] = lab[j];
    next_sentence_label[row] = swapped ? 1 : 0;
    ++row;
  }
  *mt_pos = rng.pos;
  return row;
}
