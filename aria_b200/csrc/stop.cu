// Stop strings inside the captured decode step: Hugging Face's StopStringCriteria, run on each row's history right after the
// decode advance has written the row's new token.
//
// aria_stop_check_slots: every row has its own stop set, stop ids, prompt tail and output row.
//
// A row stops when its final token completes one of its stop strings S (L bytes) in HF's sense.  For every byte prefix T0[:m]
// of the final token that ends with S's last min(m, L) bytes (m > L: S lies whole inside T0[:m], a match at once), the walk
// goes back token by token: with p bytes of S matched so far, the next token T must end with S[max(0, L - p - |T|), L - p)
// (so it may run off S's start, and an empty token always fits), then p += |T|; the row stops once p >= L.  The walk sees at
// most `lookback` tokens, the final one included: HF's window of max(len(s)) characters.  Comparing UTF-8 bytes gives HF's
// character comparison: both sides are valid UTF-8, which is self-synchronising, so a byte match of a token against a piece
// of S that starts or ends inside one of S's characters cannot be extended into a whole match.  Ids outside the vocabulary
// table match nothing; the host gives an id missing inside the table the single byte 0xFF, which no UTF-8 string holds.
#include "common.cuh"

namespace aria {

constexpr int STOP_MAX_STRINGS = 16;
constexpr int STOP_MAX_BYTES = 512;   // UTF-8 bytes of one string of at most 128 characters
constexpr int STOP_MAX_TOKENS = 128;  // lookback window and prompt tail
constexpr int STOP_MAX_IDS = 8;       // per-slot stop ids
constexpr int STOP_WARPS = 4;         // rows per CTA, one warp each
constexpr int STOP_MAX_ROWS = 1024;

struct StopVocab {
  const uint8_t* bytes;     // cleaned token strings, UTF-8, concatenated
  const int32_t* offsets;   // [V + 1]
  int32_t V;
};

__device__ __forceinline__ bool bytes_equal(const uint8_t* a, const uint8_t* b, int n) {
  for (int i = 0; i < n; ++i)
    if (a[i] != b[i]) return false;
  return true;
}

// One warp: does the history whose final token is hist(0), previous one hist(1), ... (n_hist tokens) complete one of the
// strings?  off / len: the warp's shared window (STOP_MAX_TOKENS entries each).  Same answer on every lane.
template <class Hist>
__device__ bool warp_row_stops(const StopVocab& v, const uint8_t* S_all, const int32_t* S_lens, int W, int n_hist, Hist hist,
                               int* off, int* len) {
  const int lane = threadIdx.x % 32;
  const int n_win = min(min(W, n_hist), STOP_MAX_TOKENS);
  for (int j = lane; j < n_win; j += 32) {
    const int64_t id = hist(j);
    const bool known = id >= 0 && id < v.V;
    off[j] = known ? v.offsets[id] : 0;
    len[j] = known ? v.offsets[id + 1] - v.offsets[id] : -1;
  }
  __syncwarp();
  const int len0 = n_win > 0 ? len[0] : 0;
  bool hit = false;
  if (len0 > 0) {
    const uint8_t* T0 = v.bytes + off[0];
    for (int c = lane; c < STOP_MAX_STRINGS * len0 && !hit; c += 32) {
      const int s = c / len0, m = c % len0 + 1;
      const int L = S_lens[s];
      if (L <= 0) continue;
      const uint8_t* S = S_all + s * STOP_MAX_BYTES;
      if (m >= L) {  // S whole inside T0[:m], ending at m
        hit = bytes_equal(T0 + m - L, S, L);
        continue;
      }
      if (!bytes_equal(T0, S + L - m, m)) continue;
      int p = m;
      for (int j = 1; j < n_win && p < L; ++j) {
        const int lj = len[j];
        if (lj < 0) break;
        const int k = min(lj, L - p);
        if (!bytes_equal(v.bytes + off[j] + lj - k, S + L - p - k, k)) break;
        p += lj;
      }
      hit = p >= L;
    }
  }
  const bool any = __any_sync(0xffffffffu, hit);
  return any;
}

struct SlotStopParams {
  StopVocab v;
  const uint8_t* stop_bytes;  // [R, 16, 512]
  const int32_t* stop_lens;   // [R, 16]
  const int32_t* lookback;    // [R], 0 = no strings
  const int64_t* stop_ids;    // [R, 8]
  const int32_t* n_stop_ids;  // [R]
  const int64_t* tail;        // [R, 128]
  const int32_t* tail_len;    // [R]
  const int32_t* out_tokens;  // [R, out_stride]
  int64_t out_stride;
  const int32_t* n_out;
  uint8_t* finished;
  int64_t* ids_in;
  int64_t pad;
  int32_t R;
};

__global__ void __launch_bounds__(STOP_WARPS * 32) stop_check_slots_kernel(const SlotStopParams p) {
  __shared__ int s_off[STOP_WARPS][STOP_MAX_TOKENS], s_len[STOP_WARPS][STOP_MAX_TOKENS];
  const int warp = threadIdx.x / 32;
  const int r = blockIdx.x * STOP_WARPS + warp;
  if (r >= p.R || p.finished[r]) return;  // uniform over the warp
  const int n_gen = static_cast<int>(min(static_cast<int64_t>(p.n_out[r]), p.out_stride));
  if (n_gen <= 0) return;
  const int32_t* out = p.out_tokens + r * p.out_stride;
  const int64_t* tail = p.tail + static_cast<int64_t>(r) * STOP_MAX_TOKENS;
  const auto hist = [&](int j) -> int64_t { return j < n_gen ? out[n_gen - 1 - j] : tail[STOP_MAX_TOKENS - 1 - (j - n_gen)]; };
  bool stop = false;
  const int n_ids = min(max(p.n_stop_ids[r], 0), STOP_MAX_IDS);
  for (int e = 0; e < n_ids; ++e) stop |= hist(0) == p.stop_ids[r * STOP_MAX_IDS + e];
  const int W = p.lookback[r];
  if (!stop && W > 0) {
    const int n_hist = n_gen + min(max(p.tail_len[r], 0), STOP_MAX_TOKENS);
    stop = warp_row_stops(p.v, p.stop_bytes + static_cast<int64_t>(r) * STOP_MAX_STRINGS * STOP_MAX_BYTES,
                          p.stop_lens + r * STOP_MAX_STRINGS, W, n_hist, hist, s_off[warp], s_len[warp]);
  }
  if (stop && threadIdx.x % 32 == 0) {
    p.finished[r] = 1;
    p.ids_in[r] = p.pad;  // what decode_advance_slots feeds a finished slot
  }
}

}  // namespace aria

using namespace aria;

extern "C" int aria_stop_check_slots(const uint8_t* vocab_bytes, const int32_t* vocab_offsets, int32_t V, const uint8_t* stop_bytes,
                                     const int32_t* stop_lens, const int32_t* lookback, const int64_t* stop_ids,
                                     const int32_t* n_stop_ids, const int64_t* prompt_tail, const int32_t* tail_len,
                                     const int32_t* out_tokens, int64_t out_stride, const int32_t* n_out, uint8_t* finished,
                                     int64_t* ids_in, int64_t pad_token_id, int32_t R, aria_stream_t stream_) {
  ARIA_CHECK_ARG(vocab_bytes && vocab_offsets && stop_bytes && stop_lens && lookback && stop_ids && n_stop_ids && prompt_tail);
  ARIA_CHECK_ARG(tail_len && out_tokens && n_out && finished && ids_in);
  ARIA_CHECK_ARG(V > 0 && R > 0 && R <= STOP_MAX_ROWS && out_stride > 0);
  SlotStopParams p{};
  p.v = {vocab_bytes, vocab_offsets, V};
  p.stop_bytes = stop_bytes;
  p.stop_lens = stop_lens;
  p.lookback = lookback;
  p.stop_ids = stop_ids;
  p.n_stop_ids = n_stop_ids;
  p.tail = prompt_tail;
  p.tail_len = tail_len;
  p.out_tokens = out_tokens;
  p.out_stride = out_stride;
  p.n_out = n_out;
  p.finished = finished;
  p.ids_in = ids_in;
  p.pad = pad_token_id;
  p.R = R;
  stop_check_slots_kernel<<<(R + STOP_WARPS - 1) / STOP_WARPS, STOP_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(p);
  return check_launch("stop_check_slots_kernel");
}
