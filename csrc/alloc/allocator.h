// Layer -> device allocation (the "scheduler" of the framework), C++ core.
//
// Cost model (same as the reference, scaelum/dynamics/allocator.py:104-105,310-316, plus an
// optional communication term):
//     stage_cost(d, [b, e)) = dev_time[d] * sum(layer_flops[b:e]) + cut_penalty[b] + cut_penalty[e]
//     feasible iff sum(layer_mem[b:e]) <= dev_mem[d]
// Objective: minimise the bottleneck max_d stage_cost over contiguous partitions (and, for the
// exact solver, over the order in which devices appear along the pipeline).
//
//   even_partition      == Allocator.even_allocate         (allocator.py:259-280)
//   dynamic_partition   == Allocator.dynamic_allocate      (allocator.py:181-257,295-439); `compat`
//                          reproduces the reference's greedy bit-for-bit (including its dead
//                          shrink branch), otherwise the intended two-way boundary refinement runs
//   optimal_partition   replaces the PuLP/CBC MILP of Allocator.optimal_allocate
//                          (allocator.py:25-179) with an exact solver: bisection on the bottleneck
//                          + bitmask DP over device subsets (D <= 16) / fixed-order DP otherwise.
#pragma once
#include <string>
#include <vector>

namespace sky {

struct AllocProblem {
  std::vector<double> layer_flops;  // L
  std::vector<double> layer_mem;    // L
  std::vector<double> dev_time;     // D   (relative or absolute; only ratios matter w/o penalty)
  std::vector<double> dev_mem;      // D
  std::vector<double> cut_penalty;  // L+1 or empty (cost of cutting before layer l)
};

struct AllocResult {
  std::vector<int> order;       // order[k] = device index that runs pipeline stage k
  std::vector<int> boundaries;  // D+1 monotone layer boundaries; stage k owns [b[k], b[k+1])
  double bottleneck = 0.0;
  bool exact = false;
  std::string method;
};

std::vector<int> even_partition(int num_layers, int num_devices);

// Greedy allocation in fixed device order. Throws std::runtime_error("memory allocation failed").
AllocResult dynamic_partition(const AllocProblem& p, int break_iter, bool compat);

// Exact min-max contiguous partition. `permute` lets devices take any pipeline position.
// `min_layers_per_device` is 1 for a real pipeline (every rank owns >= 1 layer).
AllocResult optimal_partition(const AllocProblem& p, bool permute, int min_layers_per_device);

double partition_bottleneck(const AllocProblem& p, const std::vector<int>& order,
                            const std::vector<int>& boundaries);

// Looped pipelines (v chunks per device, chunk k belongs to device k % D): hill-climb on the chunk
// boundaries of a partition into v * D chunks until the descending-sorted vector of per-DEVICE
// loads dev_time[d] * sum(flops of d's chunks) cannot be lowered any more (ties: the smaller most
// expensive chunk).  Every chunk keeps >= 1 unit, per-device memory caps are respected, and no
// move makes a chunk cost more than `max_chunk` (dev_time * flops; +inf: no cap) unless the
// starting partition already did.
// `p.dev_time / p.dev_mem` are per DEVICE (D entries), `boundaries` has v * D + 1 entries.
std::vector<int> refine_looped_partition(const AllocProblem& p, std::vector<int> boundaries,
                                         double max_chunk);

}  // namespace sky
