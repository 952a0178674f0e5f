// Host-side (CPU) builder of the slice x tile lists: the C-ABI counterpart of vptq_b200/lists.py for
// hosts that are not python.  Pure data layout, no GPU work; format contract in include/vptq_b200.h
// (vptq_linear_desc::lists_stream / lists_tab), consumer gemv_lists.cu.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <thread>
#include <vector>

#include "kernels.h"

namespace vptq_b200 {
namespace {

constexpr int kSlice = 4096, kTileMax = 4096, kStep = 32;

// field j of a packed row: bits [j*b, (j+1)*b) of its little-endian 32-bit word stream
inline uint32_t field_at(const uint32_t* row, int64_t words, int64_t j, int b) {
  const int64_t bit = j * b, w = bit >> 5;
  uint64_t v = row[w];
  if (w + 1 < words) v |= uint64_t(row[w + 1]) << 32;
  v >>= (bit & 31);
  return b >= 32 ? uint32_t(v) : uint32_t(v & ((uint64_t(1) << b) - 1));
}

// -------------------------------------------------------------------------------------------------------------
// Bank-aware ordering of ONE list (a pure re-ordering of its entries: the sum the decode kernel forms does not
// depend on it, its speed does).  In the kernel the 32 lanes of a warp take the 32 entries of a step; two gathers
// pay for shared-memory bank conflicts (profiles/r02_ncu_shapes_metrics.csv: 3.8 of 14.3 load wavefronts per step):
//   * the 128-bit codebook gather is conflict-free inside a quarter-warp when its 8 lanes read 8 different 16-byte
//     bank groups, i.e. hold 8 different classes (index & 7);
//   * the 16-bit x' gather is conflict-free when the 32 lanes read 32 different 4-byte banks, bank = (column >> 1) & 31.
// Per step: every class gets up to 4 slots (one per quarter; the class's entries are spread over the remaining steps),
// the slots are matched to distinct x' banks by augmenting paths (a 32 x 32 bipartite matching), unmatched slots take
// their class's fullest bank, spare lanes take entries of the fullest classes (unused banks first).  Deterministic and
// sequential; on random indices the two gathers drop from 8.6 to 7.5 wavefronts per step (the intrinsic imbalance
// of ~256 entries over 32 banks / 8 groups keeps the floor near 6.5).
// -------------------------------------------------------------------------------------------------------------
constexpr int kDealMaxEntries = 4096;
#ifndef VPTQ_DEAL_BIAS
#define VPTQ_DEAL_BIAS 0.5f
#endif
constexpr float kDealBias = VPTQ_DEAL_BIAS;
constexpr int64_t kDealChunk = 16;   // lists a worker thread takes at a time

inline int ctz32(uint32_t v) { return __builtin_ctz(v); }

void deal_list(uint32_t* entries, int n, std::vector<uint32_t>& sorted) {
  if (n < 2 || n > kDealMaxEntries) return;
  const int S = (n + kStep - 1) / kStep;
  // stable counting sort by key = class * 32 + bank
  int start[257] = {0}, cur[256];
  auto key = [](uint32_t e) { return int((e & 7u) << 5 | ((e >> 13) & 31u)); };
  for (int i = 0; i < n; ++i) ++start[key(entries[i]) + 1];
  for (int k = 0; k < 256; ++k) start[k + 1] += start[k];
  for (int k = 0; k < 256; ++k) cur[k] = start[k];
  sorted.resize(size_t(n));
  for (int i = 0; i < n; ++i) sorted[size_t(cur[key(entries[i])]++)] = entries[i];
  for (int k = 0; k < 256; ++k) cur[k] = start[k];  // pop cursor: front of every bucket
  int cnt[8], nb[32] = {0};
  int left[8][32];                                  // entries still in bucket (class, bank)
  for (int g = 0; g < 8; ++g) {
    cnt[g] = 0;
    for (int b = 0; b < 32; ++b) left[g][b] = start[g * 32 + b + 1] - start[g * 32 + b], cnt[g] += left[g][b], nb[b] += left[g][b];
  }
  int pos = 0;
  for (int s = 0; s < S; ++s) {
    const int rem = S - s, cap = s < S - 1 ? kStep : n - kStep * (S - 1);
    // how many lanes every class gets.  A quarter-warp costs one wavefront when its 8 lanes hold 8 different
    // classes and two when some class appears twice -- no matter how many do.  So the unavoidable doublings (the
    // classes are never equally full) are paid for in as few quarters as possible: a step is either all-distinct
    // (4 lanes per class) or carries `dq` "double quarters", in each of which up to 4 short classes leave a hole
    // and as many long classes appear twice.
    int want[8], tot = 0;
    if (s == S - 1) {
      for (int g = 0; g < 8; ++g) want[g] = cnt[g], tot += cnt[g];   // everything that is left (= cap)
    } else {
      int n_rem = 0;
      for (int g = 0; g < 8; ++g) n_rem += cnt[g];
      float E[8], D = 0.f, emax = 0.f;
      for (int g = 0; g < 8; ++g) {
        E[g] = float(cnt[g]) - float(n_rem) * 0.125f;
        if (E[g] > 0.f) D += E[g], emax = std::max(emax, E[g]);
      }
      const float DQ = std::max(D * 0.25f, emax);
      const int dq = std::min(4, std::max(0, int(std::ceil(DQ / float(rem) - kDealBias))));
      for (int g = 0; g < 8; ++g) want[g] = 4;
      for (int q = 0; q < dq; ++q) {
        int lo[8], hi[8];
        for (int g = 0; g < 8; ++g) lo[g] = hi[g] = g;
        std::stable_sort(lo, lo + 8, [&](int x, int y) { return E[x] < E[y]; });
        std::stable_sort(hi, hi + 8, [&](int x, int y) { return E[x] > E[y]; });
        int h = 0;
        while (h < 4 && E[lo[h]] <= -0.5f && want[lo[h]] > 0 && E[hi[h]] > 0.f && cnt[hi[h]] > want[hi[h]]) ++h;
        for (int i = 0; i < h; ++i) --want[lo[i]], E[lo[i]] += 1.f, ++want[hi[i]], E[hi[i]] -= 1.f;
      }
      for (int g = 0; g < 8; ++g) want[g] = std::min(want[g], cnt[g]), tot += want[g];
      while (tot < cap) {   // a class ran dry: its lanes go to the classes with the most entries left
        int g = 0;
        for (int c = 1; c < 8; ++c)
          if (cnt[c] - want[c] > cnt[g] - want[g]) g = c;
        if (cnt[g] <= want[g]) break;   // (cannot happen: a non-final step has >= 32 entries left)
        ++want[g], ++tot;
      }
    }
    // route the class lanes to banks: a flow classes -> buckets -> banks on 8 + 32 nodes.  Banks are served in
    // order of the entries they still hold, each up to ITS share of the remaining steps (so a heavy bank doubles
    // up early, together with the other heavy ones, instead of piling up in the last steps); what is still
    // unrouted after that raises every bank by one more, heaviest first.
    int f[8][32] = {{0}}, supply[8], used[32] = {0}, unrouted = tot;
    uint32_t resid[8];   // banks a class can still send one more entry to
    uint8_t has[32];     // classes currently routed into a bank
    for (int g = 0; g < 8; ++g) {
      supply[g] = want[g], resid[g] = 0u;
      for (int b = 0; b < 32; ++b)
        if (left[g][b] > 0) resid[g] |= 1u << b;
    }
    for (int b = 0; b < 32; ++b) has[b] = 0;
    auto augment = [&](int t) {
      // the common case: a class that still has lanes to place holds an unreserved entry of bank t (the search
      // below would return the same class: it pops the classes with lanes left first, in this order)
      for (int g = 0; g < 8; ++g)
        if (supply[g] > 0 && (resid[g] >> t & 1u)) {
          if (++f[g][t] == left[g][t]) resid[g] &= ~(1u << t);
          has[t] |= uint8_t(1u << g);
          --supply[g], ++used[t], --unrouted;
          return true;
        }
      int parent_b[32], parent_c[8], queue[8], qh = 0, qt = 0;
      uint32_t vis_b = 0u, vis_c = 0u;
      for (int g = 0; g < 8; ++g)
        if (supply[g] > 0) vis_c |= 1u << g, parent_c[g] = -1, queue[qt++] = g;
      bool found = false;
      while (qh < qt && !found) {
        const int g = queue[qh++];
        uint32_t m = resid[g] & ~vis_b;
        if (m >> t & 1u) {
          parent_b[t] = g, found = true;
          break;
        }
        for (; m; m &= m - 1) {
          const int b = ctz32(m);
          vis_b |= 1u << b, parent_b[b] = g;
          for (uint32_t cm = has[b] & ~vis_c; cm; cm &= cm - 1) {
            const int c = ctz32(cm);
            vis_c |= 1u << c, parent_c[c] = b, queue[qt++] = c;
          }
        }
      }
      if (!found) return false;
      for (int b = t;;) {
        const int g = parent_b[b];
        if (++f[g][b] == left[g][b]) resid[g] &= ~(1u << b);
        has[b] |= uint8_t(1u << g);
        const int pb = parent_c[g];
        if (pb < 0) {
          --supply[g];
          break;
        }
        if (--f[g][pb] == 0) has[pb] &= uint8_t(~(1u << g));
        resid[g] |= 1u << pb;
        b = pb;
      }
      ++used[t], --unrouted;
      return true;
    };
    int order[32];
    for (int b = 0; b < 32; ++b) order[b] = b;
    std::stable_sort(order, order + 32, [&](int x, int y) { return nb[x] > nb[y]; });
    for (int i = 0; i < 32 && unrouted > 0; ++i) {
      const int b = order[i], need = (nb[b] + rem - 1) / rem;
      for (int k = 0; k < need && unrouted > 0; ++k)
        if (!augment(b)) break;
    }
    while (unrouted > 0) {
      bool progress = false;
      for (int i = 0; i < 32 && unrouted > 0; ++i)
        if (nb[order[i]] > used[order[i]] && augment(order[i])) progress = true;
      if (!progress) break;  // cannot happen: a class with unrouted lanes has an unreserved entry in some bank
    }
    if (unrouted > 0) break;     // (defensive) give up on this list: the check after the loop restores it
    // lanes: a class's k-th entry goes to quarter k (lane 8 k + class) while k < 4; the extras fill the lanes the
    // short classes left free, from the top, so that the doubled classes share the last quarter(s)
    uint32_t lanes[32];
    bool taken[32] = {false};
    uint32_t extras[32][8];   // [k - 4][class]: a class's 5th, 6th, ... entry
    int kmax = 0;
    bool extra_set[32][8] = {{false}};
    for (int g = 0; g < 8; ++g) {
      int k = 0;
      for (int b = 0; b < 32; ++b)
        for (int j = 0; j < f[g][b]; ++j) {
          const uint32_t e = sorted[size_t(cur[g * 32 + b]++)];
          if (k < 4) lanes[k * 8 + g] = e, taken[k * 8 + g] = true;
          else extras[k - 4][g] = e, extra_set[k - 4][g] = true, kmax = std::max(kmax, k - 3);
          ++k;
        }
      for (int b = 0; b < 32; ++b) left[g][b] -= f[g][b], cnt[g] -= f[g][b], nb[b] -= f[g][b];
    }
    int lane = kStep - 1;
    for (int k = 0; k < kmax; ++k)       // all 5th entries first, then the 6th ...: one class's extras land in
      for (int g = 0; g < 8; ++g) {      // different quarters as long as the holes allow
        if (!extra_set[k][g]) continue;
        while (lane >= 0 && taken[lane]) --lane;
        if (lane < 0) break;
        lanes[lane] = extras[k][g], taken[lane] = true;
      }
    // a step's valid entries form a prefix (only the last step can be partial)
    for (int lane = 0; lane < kStep; ++lane)
      if (taken[lane]) entries[pos++] = lanes[lane];
  }
  // whatever happened above, the list must leave as a permutation of what came in
  if (pos != n) std::copy(sorted.begin(), sorted.end(), entries);
}

}  // namespace
}  // namespace vptq_b200

using namespace vptq_b200;

extern "C" int vptq_b200_lists_deal_host(uint32_t* stream_host, const uint32_t* tab_host, int64_t units, int32_t threads) {
  if (!stream_host || !tab_host || units < 0) {
    set_error("lists_deal_host: NULL argument");
    return VPTQ_ERR_INVALID;
  }
  int nt = threads > 0 ? threads : int(std::thread::hardware_concurrency());
  nt = std::max(1, std::min<int>(nt, int(std::min<int64_t>(units / kDealChunk + 1, 256))));
  std::atomic<int64_t> next{0};
  auto work = [&]() {
    std::vector<uint32_t> scratch;
    for (;;) {
      const int64_t u0 = next.fetch_add(kDealChunk);
      if (u0 >= units) break;
      for (int64_t u = u0; u < std::min<int64_t>(units, u0 + kDealChunk); ++u) {
        const uint32_t first = tab_host[u] & 0x3ffffffu, end = tab_host[u + 1] & 0x3ffffffu, tail = tab_host[u] >> 26;
        if (end <= first) continue;
        const int n = int(end - first - 1) * kStep + int(tail);
        deal_list(stream_host + size_t(first) * kStep, n, scratch);
      }
    }
  };
  if (nt == 1) {
    work();
  } else {
    std::vector<std::thread> pool;
    for (int i = 0; i < nt; ++i) pool.emplace_back(work);
    for (auto& t : pool) t.join();
  }
  return 0;
}

namespace vptq_b200 {
namespace {

// the lists of index rows of V outputs (8: include/vptq_b200.h, 16: include/vptq_b200_lists16.h); V only sets Ro
int lists_build_host(int V, const int32_t* indices_host, int64_t index_stride_row, int32_t out_features,
                     int32_t in_features, int32_t num_centroids, int32_t num_res_centroids, const uint16_t* perm_host,
                     void* stream_out, size_t stream_capacity, uint32_t* tab_out, size_t* steps_out,
                     int32_t* tile_cols_out) {
  const int K = num_centroids, Kr = num_res_centroids > 0 ? num_res_centroids : 0, I = in_features;
  if (!indices_host || !tab_out || !steps_out || !tile_cols_out || out_features < 1 || I < 8 || I > 65535) {
    set_error("lists_build_host: NULL argument or size out of range (in_features %d)", I);
    return VPTQ_ERR_INVALID;
  }
  if (K < 2 * kSlice || K % kSlice || K / kSlice > 16 || (K & (K - 1)) || Kr > 256 || (Kr & (Kr - 1))) {
    set_error("lists_build_host: needs K = NS * 4096 with 2 <= NS <= 16 and Kr <= 256 (K %d, Kr %d)", K, Kr);
    return VPTQ_ERR_UNSUPPORTED;
  }
  const int ib = ilog2(K), rb = Kr ? ilog2(Kr) : 0, b = ib + rb;
  const int NS = K / kSlice, Ro = (out_features + V - 1) / V;
  const int NT = (I + kTileMax - 1) / kTileMax, TCW = ((I + NT - 1) / NT + 7) / 8 * 8, Q = NS * NT;
  *tile_cols_out = TCW;
  const int64_t words = (int64_t(I) * b + 31) / 32;
  if (index_stride_row < words) {
    set_error("lists_build_host: index_stride_row %lld < %lld words per row", (long long)index_stride_row, (long long)words);
    return VPTQ_ERR_INVALID;
  }
  const uint32_t* base = reinterpret_cast<const uint32_t*>(indices_host);
  auto feature = [&](int c) { return perm_host ? int(perm_host[c]) : c; };
  if (perm_host)
    for (int c = 0; c < I; ++c)
      if (int(perm_host[c]) >= I) {
        set_error("lists_build_host: perm[%d] = %d is not a feature index (< %d)", c, int(perm_host[c]), I);
        return VPTQ_ERR_INVALID;
      }

  // pass 1: fields per unit -> first step and tail count of every list, combo-major
  std::vector<uint32_t> n(size_t(Q) * Ro, 0);
  for (int r = 0; r < Ro; ++r) {
    const uint32_t* row = base + int64_t(r) * index_stride_row;
    for (int c = 0; c < I; ++c) {
      const uint32_t idx = field_at(row, words, c, b) & uint32_t(K - 1);
      ++n[size_t((feature(c) / TCW) * NS + int(idx >> 12)) * Ro + r];
    }
  }
  uint64_t steps = 0;
  std::vector<uint32_t> first(n.size());
  for (size_t u = 0; u < n.size(); ++u) {
    const uint32_t st = n[u] ? (n[u] + kStep - 1) / kStep : 1u;  // every list has at least one step
    const uint32_t tail = n[u] - kStep * (st - 1);
    first[u] = uint32_t(steps);
    tab_out[u] = uint32_t(steps) | tail << 26;
    steps += st;
  }
  tab_out[n.size()] = uint32_t(steps);
  *steps_out = size_t(steps);
  if (steps >= (1ull << 26)) {
    set_error("lists_build_host: %llu steps exceed the 26-bit step counter", (unsigned long long)steps);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (!stream_out) return 0;  // sizing call
  if (stream_capacity < steps * 128) {
    set_error("lists_build_host: stream buffer of %zu bytes < %llu needed", stream_capacity, (unsigned long long)(steps * 128));
    return VPTQ_ERR_WORKSPACE;
  }

  // pass 2: zero-fill, then per row bucket the columns by (combo, bank group = index & 7) in column order
  // and deal every list out rank-major, bank-minor: 8 consecutive entries read 8 different bank groups
  uint32_t* out = static_cast<uint32_t*>(stream_out);
  std::memset(out, 0, size_t(steps) * 128);
  std::vector<std::vector<uint32_t>> bucket(size_t(Q) * 8);
  std::vector<uint32_t> fields(I);
  for (int r = 0; r < Ro; ++r) {
    const uint32_t* row = base + int64_t(r) * index_stride_row;
    for (auto& v : bucket) v.clear();
    for (int c = 0; c < I; ++c) {
      const uint32_t f = field_at(row, words, c, b);
      fields[c] = f;
      const uint32_t idx = f & uint32_t(K - 1);
      bucket[(size_t(feature(c) / TCW) * NS + (idx >> 12)) * 8 + (idx & 7)].push_back(uint32_t(c));
    }
    for (int q = 0; q < Q; ++q) {
      uint64_t pos = uint64_t(first[size_t(q) * Ro + r]) * kStep;  // entry index of the list's next slot
      size_t longest = 0;
      for (int k = 0; k < 8; ++k) longest = std::max(longest, bucket[size_t(q) * 8 + k].size());
      for (size_t rank = 0; rank < longest; ++rank)
        for (int k = 0; k < 8; ++k) {
          const std::vector<uint32_t>& bk = bucket[size_t(q) * 8 + k];
          if (rank >= bk.size()) continue;
          const uint32_t c = bk[rank], f = fields[c];
          const uint32_t lcol = uint32_t(feature(int(c)) - (q / NS) * TCW);
          out[pos++] = (f & 4095u) | lcol << 12 | (Kr ? ((f >> ib) & uint32_t(Kr - 1)) << 24 : 0u);
        }
    }
  }
  return 0;
}

}  // namespace
}  // namespace vptq_b200

extern "C" int vptq_b200_lists_build_host(const int32_t* indices_host, int64_t index_stride_row, int32_t out_features,
                                          int32_t in_features, int32_t num_centroids, int32_t num_res_centroids,
                                          const uint16_t* perm_host, void* stream_out, size_t stream_capacity,
                                          uint32_t* tab_out, size_t* steps_out, int32_t* tile_cols_out) {
  return lists_build_host(8, indices_host, index_stride_row, out_features, in_features, num_centroids,
                          num_res_centroids, perm_host, stream_out, stream_capacity, tab_out, steps_out, tile_cols_out);
}

extern "C" int vptq_b200_lists16_build_host(const int32_t* indices_host, int64_t index_stride_row, int32_t out_features,
                                            int32_t in_features, int32_t num_centroids, int32_t num_res_centroids,
                                            const uint16_t* perm_host, void* stream_out, size_t stream_capacity,
                                            uint32_t* tab_out, size_t* steps_out, int32_t* tile_cols_out) {
  return lists_build_host(16, indices_host, index_stride_row, out_features, in_features, num_centroids,
                          num_res_centroids, perm_host, stream_out, stream_capacity, tab_out, steps_out, tile_cols_out);
}
