#include "allocator.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <functional>
#include <limits>
#include <numeric>
#include <stdexcept>

namespace sky {

namespace {

struct Prefix {
  std::vector<double> flops, mem;
  explicit Prefix(const AllocProblem& p)
      : flops(p.layer_flops.size() + 1, 0.0), mem(p.layer_mem.size() + 1, 0.0) {
    for (size_t i = 0; i < p.layer_flops.size(); ++i) flops[i + 1] = flops[i] + p.layer_flops[i];
    for (size_t i = 0; i < p.layer_mem.size(); ++i) mem[i + 1] = mem[i] + p.layer_mem[i];
  }
  double f(int b, int e) const { return flops[e] - flops[b]; }
  double m(int b, int e) const { return mem[e] - mem[b]; }
};

inline double pen(const AllocProblem& p, int l) {
  if (p.cut_penalty.empty()) return 0.0;
  // no penalty at the two ends of the model (nothing is sent there)
  if (l <= 0 || l >= static_cast<int>(p.layer_flops.size())) return 0.0;
  return p.cut_penalty[l];
}

inline double stage_cost(const AllocProblem& p, const Prefix& pre, int d, int b, int e) {
  return p.dev_time[d] * pre.f(b, e) + pen(p, b) + pen(p, e);
}

void validate(const AllocProblem& p) {
  if (p.layer_flops.size() != p.layer_mem.size())
    throw std::invalid_argument("layer_flops and layer_mem must have the same length");
  if (p.dev_time.size() != p.dev_mem.size())
    throw std::invalid_argument("dev_time and dev_mem must have the same length");
  if (p.dev_time.empty()) throw std::invalid_argument("no devices");
  if (!p.cut_penalty.empty() && p.cut_penalty.size() != p.layer_flops.size() + 1)
    throw std::invalid_argument("cut_penalty must have L+1 entries");
}

}  // namespace

std::vector<int> even_partition(int L, int D) {
  if (D <= 0) throw std::invalid_argument("no devices");
  std::vector<int> b(D + 1, 0);
  const int avg = L / D;
  int rem = L - avg * D;
  for (int i = 0; i < D; ++i) {
    int n = avg;
    if (rem > 0) {
      ++n;
      --rem;
    }
    b[i + 1] = b[i] + n;
  }
  return b;
}

double partition_bottleneck(const AllocProblem& p, const std::vector<int>& order,
                            const std::vector<int>& boundaries) {
  Prefix pre(p);
  double worst = 0.0;
  for (size_t k = 0; k + 1 < boundaries.size(); ++k) {
    const int d = order.empty() ? static_cast<int>(k) : order[k];
    worst = std::max(worst, stage_cost(p, pre, d, boundaries[k], boundaries[k + 1]));
  }
  return worst;
}

// ------------------------------------------------------------------------------------------
// dynamic (greedy) allocation
// ------------------------------------------------------------------------------------------
namespace {

bool mem_ok(const std::vector<double>& avail, const std::vector<double>& used) {
  for (size_t i = 0; i < avail.size(); ++i)
    if (avail[i] < used[i]) return false;
  return true;
}

std::vector<double> span_mem(const Prefix& pre, const std::vector<int>& b) {
  std::vector<double> out(b.size() - 1);
  for (size_t j = 0; j + 1 < b.size(); ++j) out[j] = pre.m(b[j], b[j + 1]);
  return out;
}

// Memory pass: shift boundaries until every device's span fits (reference behaviour: shrink an
// over-full device from its tail, otherwise greedily pull layers forward while they fit).
void fit_memory(const AllocProblem& p, const Prefix& pre, std::vector<int>& b) {
  const int D = static_cast<int>(p.dev_time.size());
  bool satisfied = false;
  while (true) {
    std::vector<double> used = span_mem(pre, b);
    if (mem_ok(p.dev_mem, used)) {
      satisfied = true;
      break;
    }
    const std::vector<int> before = b;
    for (int j = 0; j < D - 1; ++j) {
      while (used[j] > p.dev_mem[j] && b[j + 1] - b[j] > 1) {
        --b[j + 1];
        used = span_mem(pre, b);
        if (mem_ok(p.dev_mem, used)) {
          satisfied = true;
          break;
        }
      }
      if (satisfied) break;
      while (used[j] < p.dev_mem[j] && b[j + 2] - b[j + 1] > 1) {
        const double expected = pre.m(b[j], b[j + 1] + 1);
        if (expected < p.dev_mem[j]) {
          ++b[j + 1];
          used = span_mem(pre, b);
        } else {
          break;
        }
        if (mem_ok(p.dev_mem, used)) {
          satisfied = true;
          break;
        }
      }
      if (satisfied) break;
    }
    if (satisfied || before == b) break;
  }
  if (!satisfied) throw std::runtime_error("memory allocation failed");
}

// Reference-compatible flops*time pass (allocator.py:295-368).  The "shrink" branch of the
// reference compares a quantity it calls workload_on_next_device which is in fact the CURRENT
// device's workload, so the branch never fires; compat mode keeps that.
void balance_compat(const AllocProblem& p, const Prefix& pre, std::vector<int>& b, int break_iter) {
  const int D = static_cast<int>(p.dev_time.size());
  const double tmin = *std::min_element(p.dev_time.begin(), p.dev_time.end());
  std::vector<double> t(D);
  for (int j = 0; j < D; ++j) t[j] = p.dev_time[j] / tmin;
  int iter = 0;
  while (true) {
    double total = 0.0;
    for (int j = 0; j < D; ++j) total += pre.f(b[j], b[j + 1]) * t[j];
    const double target = std::floor(total / D);
    const std::vector<int> before = b;
    for (int j = 0; j < D - 1; ++j) {
      const double cur = pre.f(b[j], b[j + 1]) * t[j];
      if (cur < target && b[j + 2] - b[j + 1] > 1) {
        if (pre.m(b[j], b[j + 1] + 1) < p.dev_mem[j]) ++b[j + 1];
      } else {
        const double last_layer = p.layer_flops[b[j + 1] - 1] * t[j];
        const double next_as_in_reference = pre.f(b[j], b[j + 1]) * t[j];
        if (next_as_in_reference < target && cur > target + last_layer && b[j + 1] - b[j] > 1) {
          if (pre.m(b[j + 1] - 1, b[j + 2]) < p.dev_mem[j + 1]) --b[j + 1];
        }
      }
    }
    if (before == b) break;
    if (++iter == break_iter) break;
  }
}

// Intended behaviour: move one layer across a boundary whenever that lowers the larger of the
// two adjacent stage costs (both directions), respecting memory.  Each accepted move strictly
// lowers the sorted cost vector, so the loop terminates.
void balance_two_way(const AllocProblem& p, const Prefix& pre, std::vector<int>& b,
                     int break_iter) {
  const int D = static_cast<int>(p.dev_time.size());
  for (int iter = 0; iter < break_iter; ++iter) {
    bool changed = false;
    for (int j = 0; j < D - 1; ++j) {
      const double cj = stage_cost(p, pre, j, b[j], b[j + 1]);
      const double cn = stage_cost(p, pre, j + 1, b[j + 1], b[j + 2]);
      const double cur = std::max(cj, cn);
      // grow j (steal first layer of j+1)
      if (b[j + 2] - b[j + 1] > 1 && pre.m(b[j], b[j + 1] + 1) <= p.dev_mem[j]) {
        const double a = stage_cost(p, pre, j, b[j], b[j + 1] + 1);
        const double c = stage_cost(p, pre, j + 1, b[j + 1] + 1, b[j + 2]);
        if (std::max(a, c) < cur * (1.0 - 1e-12)) {
          ++b[j + 1];
          changed = true;
          continue;
        }
      }
      // shrink j (push its last layer to j+1)
      if (b[j + 1] - b[j] > 1 && pre.m(b[j + 1] - 1, b[j + 2]) <= p.dev_mem[j + 1]) {
        const double a = stage_cost(p, pre, j, b[j], b[j + 1] - 1);
        const double c = stage_cost(p, pre, j + 1, b[j + 1] - 1, b[j + 2]);
        if (std::max(a, c) < cur * (1.0 - 1e-12)) {
          --b[j + 1];
          changed = true;
        }
      }
    }
    if (!changed) break;
  }
}

}  // namespace

AllocResult dynamic_partition(const AllocProblem& p, int break_iter, bool compat) {
  validate(p);
  const int L = static_cast<int>(p.layer_flops.size());
  const int D = static_cast<int>(p.dev_time.size());
  if (L < D) throw std::invalid_argument("fewer layers than devices");
  if (*std::min_element(p.dev_mem.begin(), p.dev_mem.end()) <=
      *std::min_element(p.layer_mem.begin(), p.layer_mem.end()))
    throw std::runtime_error("The smallest worker has insufficient memory for smallest layer");
  Prefix pre(p);
  std::vector<int> b = even_partition(L, D);
  fit_memory(p, pre, b);
  if (compat)
    balance_compat(p, pre, b, break_iter);
  else
    balance_two_way(p, pre, b, break_iter);
  AllocResult r;
  r.order.resize(D);
  std::iota(r.order.begin(), r.order.end(), 0);
  r.boundaries = b;
  r.bottleneck = partition_bottleneck(p, r.order, b);
  r.exact = false;
  r.method = compat ? "dynamic-compat" : "dynamic";
  return r;
}

// ------------------------------------------------------------------------------------------
// exact solver
// ------------------------------------------------------------------------------------------
namespace {

// fixed device order: classic O(D L^2) min-max DP with memory caps
bool solve_fixed_order(const AllocProblem& p, const Prefix& pre, const std::vector<int>& order,
                       int min_layers, std::vector<int>& boundaries, double& bottleneck) {
  const int L = static_cast<int>(p.layer_flops.size());
  const int D = static_cast<int>(order.size());
  const double INF = std::numeric_limits<double>::infinity();
  std::vector<std::vector<double>> best(D + 1, std::vector<double>(L + 1, INF));
  std::vector<std::vector<int>> par(D + 1, std::vector<int>(L + 1, -1));
  best[0][0] = 0.0;
  for (int k = 0; k < D; ++k) {
    const int d = order[k];
    for (int l = 0; l <= L; ++l) {
      if (best[k][l] == INF) continue;
      for (int e = l + min_layers; e <= L; ++e) {
        if (pre.m(l, e) > p.dev_mem[d]) break;
        const double c = std::max(best[k][l], stage_cost(p, pre, d, l, e));
        if (c < best[k + 1][e]) {
          best[k + 1][e] = c;
          par[k + 1][e] = l;
        }
      }
    }
  }
  if (best[D][L] == INF) return false;
  boundaries.assign(D + 1, 0);
  int pos = L;
  for (int k = D; k >= 1; --k) {
    boundaries[k] = pos;
    pos = par[k][pos];
  }
  boundaries[0] = 0;
  bottleneck = best[D][L];
  return true;
}

// feasibility of bottleneck <= T over all device orders; reach[mask] = set of layer positions
// coverable by exactly the devices in mask (each with >= min_layers layers).
struct SubsetDP {
  const AllocProblem& p;
  const Prefix& pre;
  int L, D, min_layers;
  std::vector<std::vector<uint8_t>> reach;
  std::vector<std::vector<int32_t>> parent;  // packed (d << 20 | prev_pos)

  SubsetDP(const AllocProblem& p_, const Prefix& pre_, int min_layers_)
      : p(p_), pre(pre_), L(static_cast<int>(p_.layer_flops.size())),
        D(static_cast<int>(p_.dev_time.size())), min_layers(min_layers_) {}

  // ext[d][l] = largest end e such that span [l, e) fits device d's memory and its
  // monotone cost part dev_time*flops <= T (two-pointer; non-decreasing in l)
  std::vector<std::vector<int>> ext;
  void build_ext(double T) {
    ext.assign(D, std::vector<int>(L + 1, 0));
    for (int d = 0; d < D; ++d) {
      int e = 0;
      for (int l = 0; l <= L; ++l) {
        if (e < l) e = l;
        while (e < L && pre.m(l, e + 1) <= p.dev_mem[d] && p.dev_time[d] * pre.f(l, e + 1) <= T)
          ++e;
        ext[d][l] = e;
      }
    }
  }

  bool feasible(double T, bool keep_parents) {
    const size_t nmask = static_cast<size_t>(1) << D;
    const bool has_pen = !p.cut_penalty.empty();
    build_ext(T);
    reach.assign(nmask, std::vector<uint8_t>());
    if (keep_parents) parent.assign(nmask, std::vector<int32_t>());
    reach[0].assign(L + 1, 0);
    reach[0][0] = 1;
    std::vector<int> diff(L + 2);
    for (size_t mask = 0; mask < nmask; ++mask) {
      if (reach[mask].empty()) continue;
      const std::vector<uint8_t>& cur = reach[mask];
      for (int d = 0; d < D; ++d) {
        if (mask & (static_cast<size_t>(1) << d)) continue;
        const size_t nm = mask | (static_cast<size_t>(1) << d);
        bool touched = false;
        if (!has_pen && !keep_parents) {
          std::fill(diff.begin(), diff.end(), 0);
          for (int l = 0; l + min_layers <= L; ++l) {
            if (!cur[l]) continue;
            const int lo_e = l + std::max(min_layers, 0), hi_e = ext[d][l];
            if (hi_e < lo_e) continue;
            ++diff[lo_e];
            --diff[hi_e + 1];
            touched = true;
          }
          if (!touched) continue;
          if (reach[nm].empty()) reach[nm].assign(L + 1, 0);
          int run = 0;
          for (int e = 0; e <= L; ++e) {
            run += diff[e];
            if (run > 0) reach[nm][e] = 1;
          }
        } else {
          for (int l = 0; l + min_layers <= L; ++l) {
            if (!cur[l]) continue;
            const int lo_e = l + std::max(min_layers, 0), hi_e = ext[d][l];
            for (int e = lo_e; e <= hi_e; ++e) {
              if (has_pen && stage_cost(p, pre, d, l, e) > T) continue;
              if (reach[nm].empty()) {
                reach[nm].assign(L + 1, 0);
                if (keep_parents) parent[nm].assign(L + 1, -1);
              }
              if (keep_parents && parent[nm].empty()) parent[nm].assign(L + 1, -1);
              if (!reach[nm][e]) {
                reach[nm][e] = 1;
                if (keep_parents) parent[nm][e] = (d << 20) | l;
              }
            }
          }
        }
      }
    }
    const size_t full = nmask - 1;
    return !reach[full].empty() && reach[full][L];
  }

  void extract(std::vector<int>& order, std::vector<int>& boundaries) {
    size_t mask = (static_cast<size_t>(1) << D) - 1;
    int pos = L;
    order.assign(D, 0);
    boundaries.assign(D + 1, 0);
    for (int k = D; k >= 1; --k) {
      const int32_t pk = parent[mask][pos];
      const int d = pk >> 20;
      const int prev = pk & ((1 << 20) - 1);
      order[k - 1] = d;
      boundaries[k] = pos;
      pos = prev;
      mask &= ~(static_cast<size_t>(1) << d);
    }
    boundaries[0] = 0;
  }
};

}  // namespace

AllocResult optimal_partition(const AllocProblem& p, bool permute, int min_layers) {
  validate(p);
  const int L = static_cast<int>(p.layer_flops.size());
  const int D = static_cast<int>(p.dev_time.size());
  if (min_layers < 0) min_layers = 0;
  if (L < D * min_layers) throw std::invalid_argument("fewer layers than devices");
  if (L >= (1 << 20)) throw std::invalid_argument("too many layers");
  Prefix pre(p);
  AllocResult r;
  std::vector<int> ident(D);
  std::iota(ident.begin(), ident.end(), 0);

  if (!permute || D > 10) {
    // exact for a given order; when permuting large pools, search a few orders
    std::vector<std::vector<int>> candidates{ident};
    if (permute) {
      std::vector<int> asc = ident, desc = ident;
      std::stable_sort(asc.begin(), asc.end(),
                       [&](int a, int b) { return p.dev_time[a] < p.dev_time[b]; });
      std::stable_sort(desc.begin(), desc.end(),
                       [&](int a, int b) { return p.dev_time[a] > p.dev_time[b]; });
      candidates.push_back(asc);
      candidates.push_back(desc);
    }
    bool any = false;
    for (const auto& ord : candidates) {
      std::vector<int> b;
      double bn;
      if (solve_fixed_order(p, pre, ord, min_layers, b, bn) && (!any || bn < r.bottleneck)) {
        any = true;
        r.order = ord;
        r.boundaries = b;
        r.bottleneck = bn;
      }
    }
    if (!any) throw std::runtime_error("memory allocation failed");
    if (permute) {
      // local search: adjacent swaps
      bool improved = true;
      int evals = 0;
      while (improved && evals < 64) {
        improved = false;
        for (int k = 0; k + 1 < D && evals < 64; ++k) {
          std::vector<int> ord = r.order;
          std::swap(ord[k], ord[k + 1]);
          std::vector<int> b;
          double bn;
          ++evals;
          if (solve_fixed_order(p, pre, ord, min_layers, b, bn) &&
              bn < r.bottleneck * (1.0 - 1e-12)) {
            r.order = ord;
            r.boundaries = b;
            r.bottleneck = bn;
            improved = true;
          }
        }
      }
    }
    r.exact = !permute;
    r.method = permute ? "fixed-order-dp+swap-search" : "fixed-order-dp";
    return r;
  }

  SubsetDP dp(p, pre, min_layers);
  const double INF = std::numeric_limits<double>::infinity();
  if (!dp.feasible(INF, false)) throw std::runtime_error("memory allocation failed");
  double hi = 0.0;
  {
    // any feasible solution gives an upper bound: take the fixed-order optimum if it exists,
    // else a loose bound
    std::vector<int> b;
    double bn;
    if (solve_fixed_order(p, pre, ident, min_layers, b, bn)) {
      hi = bn;
    } else {
      const double tmax = *std::max_element(p.dev_time.begin(), p.dev_time.end());
      double pmax = 0.0;
      for (double c : p.cut_penalty) pmax = std::max(pmax, c);
      hi = tmax * pre.f(0, L) + 2 * pmax;
    }
  }
  double lo = 0.0;
  for (int it = 0; it < 64 && hi - lo > 1e-12 * std::max(1.0, hi); ++it) {
    const double mid = 0.5 * (lo + hi);
    if (dp.feasible(mid, false))
      hi = mid;
    else
      lo = mid;
  }
  // hi is feasible (invariant); nudge for floating point and extract
  double T = hi * (1.0 + 1e-12) + 1e-300;
  if (!dp.feasible(T, true)) {
    T = hi * (1.0 + 1e-9);
    if (!dp.feasible(T, true)) throw std::runtime_error("exact solver lost feasibility");
  }
  dp.extract(r.order, r.boundaries);
  r.bottleneck = partition_bottleneck(p, r.order, r.boundaries);
  r.exact = true;
  r.method = "bisection+subset-dp";
  return r;
}

// ------------------------------------------------------------------------------------------
// looped pipelines: balance the per-device sums of a chunk-level partition
// ------------------------------------------------------------------------------------------
namespace {
struct LoopedScore {
  std::vector<double> sorted_loads;  // descending
  double worst_chunk = 0.0;
  std::vector<double> loads;         // per device, unsorted
  bool feasible = true;
  bool better_than(const LoopedScore& o) const {
    if (sorted_loads != o.sorted_loads)
      return std::lexicographical_compare(sorted_loads.begin(), sorted_loads.end(),
                                          o.sorted_loads.begin(), o.sorted_loads.end());
    return worst_chunk < o.worst_chunk;
  }
};

LoopedScore looped_score(const std::vector<double>& pre_f, const std::vector<double>& pre_m,
                         const AllocProblem& p, const std::vector<int>& b) {
  const int D = static_cast<int>(p.dev_time.size());
  const int VP = static_cast<int>(b.size()) - 1;
  LoopedScore s;
  s.loads.assign(D, 0.0);
  std::vector<double> mem(D, 0.0);
  for (int k = 0; k < VP; ++k) {
    const double c = (pre_f[b[k + 1]] - pre_f[b[k]]) * p.dev_time[k % D];
    s.loads[k % D] += c;
    mem[k % D] += pre_m[b[k + 1]] - pre_m[b[k]];
    s.worst_chunk = std::max(s.worst_chunk, c);
  }
  for (int d = 0; d < D; ++d)
    if (mem[d] > p.dev_mem[d]) s.feasible = false;
  s.sorted_loads = s.loads;
  std::sort(s.sorted_loads.begin(), s.sorted_loads.end(), std::greater<double>());
  return s;
}
}  // namespace

std::vector<int> refine_looped_partition(const AllocProblem& p, std::vector<int> b,
                                         double max_chunk) {
  const int D = static_cast<int>(p.dev_time.size());
  const int VP = static_cast<int>(b.size()) - 1;
  const int L = static_cast<int>(p.layer_flops.size());
  if (D <= 0 || VP <= 0 || VP % D != 0 || b.front() != 0 || b.back() != L)
    throw std::invalid_argument("refine_looped_partition: boundaries do not describe v * D chunks");
  std::vector<double> pre_f(L + 1, 0.0), pre_m(L + 1, 0.0);
  for (int i = 0; i < L; ++i) {
    pre_f[i + 1] = pre_f[i] + p.layer_flops[i];
    pre_m[i + 1] = pre_m[i] + p.layer_mem[i];
  }
  LoopedScore cur = looped_score(pre_f, pre_m, p, b);
  // a start that is already over the cap may keep its worst chunk, but no move may raise it
  const double cap = std::max(max_chunk, cur.worst_chunk);
  for (int iter = 0; iter < 20 * VP; ++iter) {
    int busiest = 0;
    for (int d = 1; d < D; ++d)
      if (cur.loads[d] > cur.loads[busiest]) busiest = d;
    bool found = false;
    LoopedScore best;
    std::vector<int> best_b;
    for (int k = busiest; k < VP; k += D) {
      for (int side = 0; side < 2; ++side) {
        if (b[k + 1] - b[k] <= 1) continue;
        std::vector<int> nb = b;
        if (side == 0 && k > 0)
          nb[k] += 1;            // first unit of chunk k goes to chunk k - 1
        else if (side == 1 && k < VP - 1)
          nb[k + 1] -= 1;        // last unit of chunk k goes to chunk k + 1
        else
          continue;
        LoopedScore sc = looped_score(pre_f, pre_m, p, nb);
        if (sc.feasible && sc.worst_chunk <= cap && sc.better_than(cur) &&
            (!found || sc.better_than(best))) {
          best = sc;
          best_b = nb;
          found = true;
        }
      }
    }
    if (!found) break;
    cur = best;
    b = best_b;
  }
  return b;
}

}  // namespace sky
