// oracle/ref_replay.cpp — TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// Compiled with the unmodified reference sources and `-include replay_rng.h` by oracle/Makefile
// into oracle/_ref/libyttm_ref_replay.so: the reference's own BPE-dropout (DropoutQueue and the
// caller's loop, bpe.cpp:1417-1453 and 1549-1589) fed with the product's Philox draws.
//
// The product keys the draws of a word by (seed, sentence index, byte offset of the word in its
// sentence).  encode_sentence treats the words of a sentence independently, so the reference is
// run one word at a time: the key is set, the word's bytes go through encode_as_ids (n_threads = 1,
// so on this thread) and, on request, through encode_as_subwords with the key set again.  Both
// calls must use the same number of draws.  <BOS>, <EOS> and reverse are applied by the caller.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "bpe.h"

namespace {
void set_err(char *err, int errlen, const std::string &m) {
  if (err && errlen > 0) {
    std::strncpy(err, m.c_str(), errlen - 1);
    err[errlen - 1] = 0;
  }
}
struct Replay {
  vkcom::BaseEncoder *enc = nullptr;
  std::vector<int32_t> ids;
  std::vector<uint64_t> id_offs;
  std::vector<uint32_t> draws;
  std::string text;  // pieces: '\x01' between the pieces of a word, '\n' after each word
};
}  // namespace

extern "C" {

void *rpl_open(const char *model_path, char *err, int errlen) {
  vkcom::Status st;
  auto *h = new Replay();
  h->enc = new vkcom::BaseEncoder(std::string(model_path), 1, &st);
  if (!st.ok()) {
    set_err(err, errlen, st.message);
    delete h->enc;
    delete h;
    return nullptr;
  }
  return h;
}

void rpl_close(void *hv) {
  auto *h = static_cast<Replay *>(hv);
  if (!h) return;
  delete h->enc;
  delete h;
}

// Word i = bytes[offs[i], offs[i+1]) with key (seed[i], sent[i], word_off[i]).  Results stay in the
// handle (rpl_result); *n_ids and *n_text give their sizes.  Returns 0, or 1 with a message.
int rpl_encode(void *hv, const char *bytes, const uint64_t *offs, uint64_t n_words, const uint64_t *seed,
               const uint64_t *sent, const uint32_t *word_off, double p, int subwords, uint64_t *n_ids,
               uint64_t *n_text, char *err, int errlen) {
  auto *h = static_cast<Replay *>(hv);
  h->ids.clear(); h->id_offs.assign(1, 0); h->draws.clear(); h->text.clear();
  for (uint64_t i = 0; i < n_words; i++) {
    std::vector<std::string> w(1, std::string(bytes + offs[i], bytes + offs[i + 1]));
    std::vector<std::vector<int>> ids;
    yttm_replay::set_key(seed[i], sent[i], word_off[i]);
    vkcom::Status st = h->enc->encode_as_ids(w, &ids, false, false, false, p);
    if (!st.ok()) { set_err(err, errlen, st.message); return 1; }
    const yttm_replay::Key k = yttm_replay::key();
    if (k.calls != 2ull * k.draw) { set_err(err, errlen, "an engine word outside a two-word draw"); return 1; }
    for (int v : ids[0]) h->ids.push_back(v);
    h->id_offs.push_back(h->ids.size());
    h->draws.push_back(k.draw);
    if (subwords) {
      std::vector<std::vector<std::string>> pieces;
      yttm_replay::set_key(seed[i], sent[i], word_off[i]);
      st = h->enc->encode_as_subwords(w, &pieces, false, false, false, p);
      if (!st.ok()) { set_err(err, errlen, st.message); return 1; }
      if (yttm_replay::key().draw != k.draw || pieces[0].size() != ids[0].size()) {
        set_err(err, errlen, "encode_as_subwords replayed differently from encode_as_ids");
        return 1;
      }
      for (size_t j = 0; j < pieces[0].size(); j++) {
        if (j) h->text.push_back('\x01');
        h->text += pieces[0][j];
      }
      h->text.push_back('\n');
    }
  }
  *n_ids = h->ids.size();
  *n_text = h->text.size();
  return 0;
}

// ids: n_ids entries, id_offs / draws: n_words + 1 / n_words entries, text: n_text bytes.
void rpl_result(void *hv, int32_t *ids, uint64_t *id_offs, uint32_t *draws, char *text) {
  auto *h = static_cast<Replay *>(hv);
  std::memcpy(ids, h->ids.data(), h->ids.size() * sizeof(int32_t));
  std::memcpy(id_offs, h->id_offs.data(), h->id_offs.size() * sizeof(uint64_t));
  std::memcpy(draws, h->draws.data(), h->draws.size() * sizeof(uint32_t));
  std::memcpy(text, h->text.data(), h->text.size());
}

// The engine as the reference sees it, under key (seed, sent, word_off): words[0..2n) are its raw
// output and canon[0..n) what uniform_real_distribution<>(0, 1) makes of the same stream.
void rpl_engine(uint64_t seed, uint64_t sent, uint32_t word_off, uint32_t n, uint32_t *words, double *canon) {
  std::mt19937 g;  // the replay engine, like the reference's `rnd`
  std::uniform_real_distribution<> dist(0, 1);
  yttm_replay::set_key(seed, sent, word_off);
  for (uint32_t i = 0; i < n; i++) canon[i] = dist(g);
  yttm_replay::set_key(seed, sent, word_off);
  for (uint32_t i = 0; i < 2 * n; i++) words[i] = g();
}

}  // extern "C"
