// Host-side property test of the exclusion-cache rule the device-resident ICP loop runs (cilantro_b200/csrc/cache_rule.hpp
// is the SAME source the cached-pass kernel compiles; here it is compiled for the host, directed rounding through
// <cfenv>). A brute-force search with the contract arithmetic plays the search kernel and hands the rule the TIGHTEST
// valid exclusion radius (the computed distance of the second-nearest point); over a converging sequence of transforms
// every verdict of the rule is compared with a fresh brute-force search:
//   hit + pair  -> brute force returns the same index and the same d2 bits, strictly unique, inside the radius
//   hit, no pair-> brute force finds nothing inside the radius
// and the run must not be vacuous (most queries hit in the late iterations). The same harness with the radius inflated
// by 50 % must REPORT violations (the test has teeth).
// Build: g++ -std=c++17 -O2 -frounding-math -ffp-contract=off -I cilantro_b200/csrc tests/cpp/test_cache_rule.cpp
#include "cache_rule.hpp"

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

namespace {

struct Rigid {
  float r[9];
  float t[3];
};
struct P3 {
  float x, y, z;
};

uint32_t bits(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return u;
}

Rigid pose(const double axis_in[3], double angle, const double t[3]) {
  double a[3] = {axis_in[0], axis_in[1], axis_in[2]};
  const double n = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  for (double& v : a) v /= n;
  const double c = std::cos(angle), s = std::sin(angle), C = 1 - c;
  const double R[9] = {c + a[0] * a[0] * C,        a[0] * a[1] * C - a[2] * s, a[0] * a[2] * C + a[1] * s,
                       a[1] * a[0] * C + a[2] * s, c + a[1] * a[1] * C,        a[1] * a[2] * C - a[0] * s,
                       a[2] * a[0] * C - a[1] * s, a[2] * a[1] * C + a[0] * s, c + a[2] * a[2] * C};
  Rigid T;
  for (int i = 0; i < 9; i++) T.r[i] = (float)R[i];
  for (int i = 0; i < 3; i++) T.t[i] = (float)t[i];
  return T;
}

struct Found {
  int idx;       // nearest point with d2 < max_d2 (lowest index on ties), -1 = none
  float d2;      // its computed squared distance
  float D2;      // computed squared distance of the nearest OTHER point (all points when idx = -1)
  bool unique;   // no other point has a computed d2 <= d2
};

// the search kernel's answer, by brute force with the contract arithmetic (nn_search.cuh: accept iff d2 < max_d2,
// exact ties -> lowest index)
Found brute(const std::vector<P3>& dst, const Rigid& T, const P3& s, float max_d2) {
  float qx, qy, qz;
  cb::rule::transform_point(T, s.x, s.y, s.z, qx, qy, qz);
  float b1 = INFINITY, b2 = INFINITY;
  int i1 = -1;
  for (size_t j = 0; j < dst.size(); j++) {
    const float d2 = cb::rule::contract_d2(qx, qy, qz, dst[j].x, dst[j].y, dst[j].z);
    if (d2 < b1) {
      b2 = b1;
      b1 = d2;
      i1 = (int)j;
    } else if (d2 < b2) {
      b2 = d2;
    }
  }
  Found f;
  if (b1 < max_d2) {
    f.idx = i1;
    f.d2 = b1;
    f.D2 = b2;
    f.unique = b2 > b1;
  } else {
    f.idx = -1;
    f.d2 = max_d2;
    f.D2 = b1;  // every point is at least this far away
    f.unique = true;
  }
  return f;
}

struct Stats {
  long hits_pair = 0, hits_empty = 0, misses = 0, violations = 0;
  long last_hits = 0, last_total = 0;
};

// lattice = true: the destination points sit on a regular lattice (spacing 1/16) and a third of the source points on
// its cell centres / face centres / edge midpoints, i.e. exactly equidistant from 8 / 4 / 2 lattice points: exact ties
// of the computed distances, which must never come out as cached pairs.
Stats run(int n_dst, int n_src, float max_d2, double radius_scale, uint32_t seed, int iterations, bool lattice = false) {
  std::mt19937 rng(seed);
  std::uniform_real_distribution<float> uni(0.f, 1.f), jit(-0.002f, 0.002f);
  std::vector<P3> dst(n_dst), src(n_src);
  for (auto& p : dst) p = {uni(rng), uni(rng), uni(rng)};
  if (lattice) {
    int side = 1;
    while ((side + 1) * (side + 1) * (side + 1) <= n_dst) side++;
    n_dst = side * side * side;
    dst.resize(n_dst);
    for (int j = 0; j < n_dst; j++)
      dst[j] = {(j % side) * 0.0625f, ((j / side) % side) * 0.0625f, (j / (side * side)) * 0.0625f};
  }
  // source points = destination points (some of them displaced beyond the radius) seen from a different pose
  const double ax0[3] = {0.3, -0.5, 0.81}, t0[3] = {0.01, -0.02, 0.015};
  const Rigid Tgen = pose(ax0, 0.03, t0);
  for (int i = 0; i < n_src; i++) {
    P3 p = dst[i % n_dst];
    p.x += jit(rng), p.y += jit(rng), p.z += jit(rng);
    if (i % 7 == 3) p.x += 0.5f;  // outliers: nothing inside the correspondence radius
    float x, y, z;
    cb::rule::transform_point(Tgen, p.x, p.y, p.z, x, y, z);
    src[i] = {x, y, z};
    if (lattice && i % 3 == 0) {  // exactly between lattice points; not moved by Tgen, the identity is among the transforms
      const P3 b = dst[i % n_dst];
      const int kind = (i / 3) % 3;
      src[i] = {b.x + 0.03125f, b.y + (kind < 2 ? 0.03125f : 0.f), b.z + (kind < 1 ? 0.03125f : 0.f)};
    }
  }
  // a converging sequence of transforms around the inverse pose: the update shrinks geometrically, like ICP's
  std::vector<Rigid> Ts;
  if (lattice) {  // two identical identity transforms first: the tie queries are evaluated exactly on their ties
    const double axz[3] = {0, 0, 1}, tz[3] = {0, 0, 0};
    Ts.push_back(pose(axz, 0.0, tz));
    Ts.push_back(pose(axz, 0.0, tz));
    iterations += 2;
  }
  for (int k = 0; (int)Ts.size() <= iterations; k++) {
    const double sc = std::pow(0.45, k);
    const double ax[3] = {-0.3 + 0.2 * sc, 0.5, -0.81 + 0.1 * sc};
    const double t[3] = {-0.01 + 0.004 * sc, 0.02 - 0.003 * sc, -0.015 + 0.002 * sc};
    Ts.push_back(pose(ax, 0.03 + 0.01 * sc, t));
  }
  std::vector<int> seedv(n_src);
  std::vector<float> rad(n_src);
  auto search = [&](int i, const Rigid& T) {
    const Found f = brute(dst, T, src[i], max_d2);
    seedv[i] = f.idx;
    rad[i] = (float)(radius_scale * cb::rule::cache_radius(f.D2));
  };
  for (int i = 0; i < n_src; i++) search(i, Ts[0]);
  Stats st;
  for (int k = 1; k <= iterations; k++) {
    long hits = 0;
    for (int i = 0; i < n_src; i++) {
      bool miss = true;
      if (rad[i] > 0.f) {
        cb::rule::Verdict v;
        P3 p{0.f, 0.f, 0.f};
        const int sd = seedv[i];
        cb::rule::cached_match_test(Ts[k], Ts[k - 1], src[i].x, src[i].y, src[i].z, rad[i], sd, max_d2,
                                    [&] { return dst[sd]; }, p, v);
        miss = v.miss;
        if (!miss) {
          const Found f = brute(dst, Ts[k], src[i], max_d2);
          bool ok;
          if (v.pair) {
            ok = f.idx == sd && bits(f.d2) == bits(v.d2) && f.unique && v.d2 < max_d2;
            st.hits_pair++;
          } else {
            ok = f.idx == -1;
            st.hits_empty++;
          }
          if (!ok) {
            if (st.violations < 5)
              std::printf("  violation: iteration %d query %d cached %d pair %d d2 %.9g | brute %d d2 %.9g unique %d\n", k, i, sd,
                          (int)v.pair, v.d2, f.idx, f.d2, (int)f.unique);
            st.violations++;
          }
          rad[i] = v.r2;
          hits++;
        }
      }
      if (miss) {
        st.misses++;
        search(i, Ts[k]);
      }
    }
    st.last_hits = hits;
    st.last_total = n_src;
  }
  return st;
}

int check(bool cond, const char* what) {
  std::printf("%s  %s\n", cond ? "ok  " : "FAIL", what);
  return cond ? 0 : 1;
}

// hand-made cases around the strict comparisons
int edge_cases() {
  int bad = 0;
  const double ax[3] = {0, 0, 1}, t0[3] = {0, 0, 0};
  const Rigid I = pose(ax, 0.0, t0);
  cb::rule::Verdict v;
  P3 p{0, 0, 0};
  const P3 m{0.25f, 0.f, 0.f};
  // no motion, match at distance 0.25, every other point at >= 0.25 (an exact tie of the two nearest): never a hit
  cb::rule::cached_match_test(I, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.0625f), 0, 1.f, [&] { return m; }, p, v);
  bad += check(v.miss, "exact tie between the match and the second-nearest point is searched again");
  // second-nearest clearly farther: hit, d2 is the contract value, radius unchanged without motion
  cb::rule::cached_match_test(I, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.09f), 0, 1.f, [&] { return m; }, p, v);
  bad += check(!v.miss && v.pair && bits(v.d2) == bits(0.0625f) && v.r2 == cb::rule::cache_radius(0.09f),
               "clear second-nearest: hit with the contract d2");
  // the match outside the correspondence radius, everything else farther than the radius: hit without a pair
  cb::rule::cached_match_test(I, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.09f), 0, 0.05f, [&] { return m; }, p, v);
  bad += check(!v.miss && !v.pair, "match outside the radius and nothing else inside: no correspondence, no search");
  // ... but not when another point may be inside the radius
  cb::rule::cached_match_test(I, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.04f), 0, 0.05f, [&] { return m; }, p, v);
  bad += check(v.miss, "match outside the radius, another point possibly inside: searched again");
  // nothing cached inside the radius: stays empty only while the bound covers the radius
  cb::rule::cached_match_test(I, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.09f), -1, 0.05f, [&] { return m; }, p, v);
  bad += check(!v.miss && !v.pair, "empty neighbourhood stays empty while max_d2 <= lim");
  cb::rule::cached_match_test(I, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.05f), -1, 0.05f, [&] { return m; }, p, v);
  bad += check(v.miss, "max_d2 equal to the bound before the margins: searched again");
  // a motion larger than the radius: searched again, nothing stored
  const double tbig[3] = {0.5, 0, 0};
  const Rigid Tm = pose(ax, 0.0, tbig);
  cb::rule::cached_match_test(Tm, I, 0.f, 0.f, 0.f, cb::rule::cache_radius(0.09f), 0, 1.f, [&] { return m; }, p, v);
  bad += check(v.miss && v.r2 == 0.f, "motion beyond the radius: searched again");
  // the radius shrinks by at least the motion
  const double tsm[3] = {0.01, 0, 0};
  const Rigid Ts = pose(ax, 0.0, tsm);
  cb::rule::cached_match_test(Ts, I, 0.f, 0.f, 0.f, 0.3f, 0, 1.f, [&] { return m; }, p, v);
  bad += check(!v.miss && v.r2 < 0.3f - 0.01f && v.r2 > 0.3f - 0.0101f, "radius shrinks by the (rounded-up) motion");
  // unknown bound (D2 = 0) caches nothing
  bad += check(cb::rule::cache_radius(0.f) == 0.f && cb::rule::cache_radius(0.09f) < std::sqrt(0.09f),
               "cache_radius rounds down; an unknown bound caches nothing");
  return bad;
}

}  // namespace

int main() {
  int bad = edge_cases();
  struct Case {
    int n_dst, n_src;
    float max_d2;
    uint32_t seed;
  };
  const Case cases[] = {{3000, 3000, 0.02f * 0.02f, 1u}, {3000, 2000, 0.2f * 0.2f, 2u}, {1500, 3000, 0.005f * 0.005f, 3u}};
  for (const Case& c : cases) {
    const Stats s = run(c.n_dst, c.n_src, c.max_d2, 1.0, c.seed, 7);
    std::printf("n_dst %d n_src %d max_d2 %.3g: %ld pair hits, %ld empty hits, %ld searches, %ld violations; last iteration %ld of %ld cached\n",
                c.n_dst, c.n_src, c.max_d2, s.hits_pair, s.hits_empty, s.misses, s.violations, s.last_hits, s.last_total);
    bad += check(s.violations == 0, "every cached verdict equals a fresh exact search");
    bad += check(s.hits_pair + s.hits_empty > 4 * (long)c.n_src && 10 * s.last_hits > 9 * s.last_total,
                 "the run is not vacuous (most queries cached by the last iteration)");
  }
  {
    const Stats s = run(4096, 4000, 0.05f * 0.05f, 1.0, 5u, 6, true);
    std::printf("lattice (exact ties): %ld pair hits, %ld empty hits, %ld searches, %ld violations\n", s.hits_pair, s.hits_empty,
                s.misses, s.violations);
    bad += check(s.violations == 0, "lattice with exact ties: every cached verdict equals a fresh exact search");
  }
  // the harness has teeth: an exclusion radius 50 % too large must be caught
  const Stats t = run(3000, 3000, 0.2f * 0.2f, 1.5, 4u, 4);
  std::printf("radius inflated x1.5: %ld violations\n", t.violations);
  bad += check(t.violations > 0, "an invalid (inflated) radius is detected by the same harness");
  if (bad == 0) std::printf("all cache-rule checks passed\n");
  return bad ? 1 : 0;
}
