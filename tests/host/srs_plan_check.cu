// Host-only check (built by nvcc, runs without a GPU) of the sparse-sum planner of groth16_b200/csrc/srs.cuh (SrsSumPlan,
// srs_split): for column lengths 0, 1, 16, 17, 16^k + 1 and mixed layouts, at chunk sizes 2, 3 and 16, every level's chunks
// cover the items of that level once, in order, hold at most `k` items and never cross a segment, and the last level leaves
// exactly one item in every non-empty column and none in an empty one.  The plan is also run on integers standing for points:
// every column's final item must be the sum of its entries.
#include <cstdio>
#include <vector>
#include "../../groth16_b200/csrc/srs.cuh"
using namespace g16;

static int bad = 0, cases = 0;
#define CHECK(cond, ...)            \
  do {                              \
    cases++;                        \
    if (!(cond)) {                  \
      bad++;                        \
      fprintf(stderr, __VA_ARGS__); \
      fprintf(stderr, "\n");        \
    }                               \
  } while (0)

static void check(const std::vector<uint64_t>& lens, uint32_t k) {
  std::vector<uint64_t> cp(1, 0);
  for (uint64_t l : lens) cp.push_back(cp.back() + l);
  SrsSumPlan plan;
  plan.make(cp, k);
  // items of level 0: entry e stands for the value e + 1; the reduction adds chunk by chunk as srs_reduce_kernel does
  std::vector<uint64_t> items(cp.back());
  for (uint64_t e = 0; e < items.size(); e++) items[e] = e + 1;
  std::vector<uint64_t> seg = cp;
  for (const std::vector<uint64_t>& lv : plan.levels) {
    CHECK(!lv.empty() && lv.front() == 0 && lv.back() == items.size(), "level does not cover its items");
    std::vector<uint64_t> out(lv.size() - 1), next(seg.size(), 0);
    size_t s = 0;
    for (size_t c = 0; c + 1 < lv.size(); c++) {
      CHECK(lv[c] < lv[c + 1] && lv[c + 1] - lv[c] <= k, "chunk %zu: empty or longer than %u", c, k);
      while (s + 1 < seg.size() && seg[s + 1] <= lv[c]) s++;
      CHECK(lv[c] >= seg[s] && lv[c + 1] <= seg[s + 1], "chunk %zu crosses a segment", c);
      for (uint64_t j = lv[c]; j < lv[c + 1]; j++) out[c] += items[j];
    }
    items.swap(out);
    // segments of the next level: chunk counts per segment, as srs_split reports them
    std::vector<uint64_t> nseg(1, 0);
    size_t c = 0;
    for (size_t t = 0; t + 1 < seg.size(); t++) {
      while (c + 1 < lv.size() && lv[c] < seg[t + 1]) c++;
      nseg.push_back(c);
    }
    seg.swap(nseg);
  }
  CHECK(plan.last == seg, "final segment pointers differ from the walk");
  for (size_t j = 0; j < lens.size(); j++) {
    const uint64_t have = plan.last[j + 1] - plan.last[j];
    CHECK(have == (lens[j] ? 1u : 0u), "column %zu of length %llu ends with %llu items", j, (unsigned long long)lens[j],
          (unsigned long long)have);
    if (have == 1) {
      uint64_t want = 0;
      for (uint64_t e = cp[j]; e < cp[j + 1]; e++) want += e + 1;
      CHECK(items[plan.last[j]] == want, "column %zu sums to the wrong value", j);
    }
  }
}

int main() {
  const std::vector<std::vector<uint64_t>> layouts = {
      {}, {0}, {1}, {16}, {17}, {0, 0, 0}, {1, 0, 16, 17, 0, 2},
      {4097}, {65537, 0, 3}, {256, 257, 255, 1, 0, 4096}, {1048577, 5, 0}};
  for (uint32_t k : {2u, 3u, SRS_CHUNK})
    for (const auto& l : layouts) check(l, k);
  printf("srs planner: %d checks, %d mismatches\n", cases, bad);
  return bad ? 1 : 0;
}
