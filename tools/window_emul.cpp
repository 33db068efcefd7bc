// tools/window_emul.cpp -- TEST/DEVELOPMENT INFRASTRUCTURE.
// Host emulation of the window-based parse kernels (fixed G positions resolved per window with the distance cache of the
// window start, then the straight-line greedy / lazy walk).  Used to check, without a GPU, that the windowed formulation
// with G = 2 (k_parse_pair: four parse units per warp) and G = 8 (parse_unit_warp4: one per warp) produces exactly the
// commands of the sequential specification parse_range() of bro_parse.cuh.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "bro_common.cuh"
#include "bro_parse.cuh"
using namespace bro;

template <int G>
static uint32_t parse_range_windowed(const EncParams& P, const uint8_t* data, const uint32_t* best, uint32_t rstart, uint32_t rend,
                                     RawCmd* out, uint32_t* tail, uint32_t* ncopy, bool D, int32_t* dc, uint64_t* nwin) {
  const uint32_t htl = P.hash_type == 6 ? 8u : 4u;
  const uint32_t window = P.quality < 9 ? 64u : 512u;
  const uint32_t uend = rend;
  uint32_t pos = rstart, insert_len = 0, ncmd = 0, copied = 0, arh = pos + window;
  bool have_m = false;
  uint32_t m_len = 0, m_dist = 0, m_score = 0;
  int delayed = 0;
  while (have_m || pos + htl < uend) {
    ++*nwin;
    const uint32_t wbase = pos;
    Match res[G];
    bool fnd[G];
    uint32_t found = 0;
    for (int j = 0; j < G; ++j) {
      const uint32_t p = wbase + j;
      fnd[j] = false;
      if (p < uend) fnd[j] = find_match(P, data, best, dc, p, uend - p, &res[j], D);
      if (fnd[j]) found |= 1u << j;
    }
    // ---- straight-line phase B ----
    bool wdone = false, accept = false;
    uint32_t j = 0;
    {
      const bool doA = !have_m;
      const uint32_t lim = bmin((uint32_t)G, uend - htl - wbase);
      const uint32_t cand = found & (lim >= 32 ? 0xFFFFFFFFu : ((1u << lim) - 1u));
      const uint32_t f = cand ? (uint32_t)__builtin_ctz(cand) : lim;
      const uint32_t run = f;
      uint32_t steps = run;
      bool jump = false;
      if (run > 0 && pos + run > arh) { steps = pos > arh ? 1u : (arh - pos + 1u); jump = true; }
      if (doA) { insert_len += steps; pos += steps; j = steps; }
      if (doA && jump) {
        const uint32_t margin = bmax(htl - 1u, 4u);
        if (pos + 16 + margin >= uend) { insert_len += uend - pos; pos = uend; }
        else if (pos > arh + 4 * window) { insert_len += 16; pos += 16; }
        else { insert_len += 8; pos += 8; }
        wdone = true;
      } else if (doA && (!cand || j >= (uint32_t)G)) wdone = true;
      else if (doA) { m_len = res[j].len; m_dist = res[j].dist; m_score = res[j].score; have_m = true; delayed = 0; }
    }
    for (int s = 0; s < G - 1; ++s) {
      const bool doB = !wdone && !accept && have_m;
      if (doB && j + 1 >= (uint32_t)G) wdone = true;
      else if (doB) {
        const bool f2 = (found >> (j + 1)) & 1u;
        if (f2 && res[j + 1].score >= m_score + 175u) {
          pos++; insert_len++; j++;
          m_len = res[j].len; m_dist = res[j].dist; m_score = res[j].score;
          if (!(++delayed < 4 && pos + htl < uend)) accept = true;
        } else accept = true;
      }
    }
    if (!wdone && !accept && have_m && G == 1) accept = true;
    if (accept) {
      const uint32_t mb = len_bytes(m_len);
      arh = pos + 2 * mb + window;
      if (!len_is_dict(m_len) && (int32_t)m_dist != dc[0]) { dc[3] = dc[2]; dc[2] = dc[1]; dc[1] = dc[0]; dc[0] = (int32_t)m_dist; }
      if (out) { out[ncmd].insert_len = insert_len; out[ncmd].copy_len = m_len; out[ncmd].distance = m_dist; }
      ++ncmd;
      insert_len = 0;
      copied += mb;
      pos += mb;
      have_m = false;
    }
  }
  insert_len += uend - pos;
  *tail = insert_len;
  *ncopy = copied;
  return ncmd;
}

extern "C" int window_emul_check(const EncParams* Pin, const uint8_t* data, const uint32_t* best, uint32_t n, uint64_t* win2, uint64_t* win8) {
  EncParams P = *Pin;
  const uint32_t CU = P.unit / 2 + 2;
  std::vector<RawCmd> a(CU), b(CU), c(CU);
  int bad = 0;
  for (uint32_t s = 0; s < n; s += P.unit) {
    const uint32_t e = bmin(n, s + P.unit);
    int32_t d0[4] = {0x3fffffff, 0x3fffffff, 0x3fffffff, 0x3fffffff}, d1[4], d2[4];
    memcpy(d1, d0, 16); memcpy(d2, d0, 16);
    uint32_t t0, c0, t1, c1, t2, c2;
    auto find = [&](uint32_t p, uint32_t max_len, Match* m) { return find_match(P, data, best, d0, p, max_len, m, P.use_dict != 0); };
    auto store = [&](uint32_t k, uint32_t ins, uint32_t len, uint32_t dist) { a[k] = RawCmd{ins, len, dist}; };
    uint32_t n0 = parse_range(P, s, e, d0, find, store, &t0, &c0);
    uint32_t n1 = parse_range_windowed<2>(P, data, best, s, e, b.data(), &t1, &c1, P.use_dict != 0, d1, win2);
    uint32_t n2 = parse_range_windowed<8>(P, data, best, s, e, c.data(), &t2, &c2, P.use_dict != 0, d2, win8);
    if (n0 != n1 || n0 != n2 || t0 != t1 || t0 != t2 || c0 != c1 || c0 != c2 || memcmp(a.data(), b.data(), n0 * sizeof(RawCmd)) ||
        memcmp(a.data(), c.data(), n0 * sizeof(RawCmd)) || memcmp(d0, d1, 16) || memcmp(d0, d2, 16)) {
      if (bad < 5) fprintf(stderr, "unit at %u differs: n %u %u %u tail %u %u %u\n", s, n0, n1, n2, t0, t1, t2);
      ++bad;
    }
  }
  return bad;
}
