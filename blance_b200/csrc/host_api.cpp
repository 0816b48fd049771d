// blance_b200/csrc/host_api.cpp — see host_api.hpp.  Interning (strings -> flat
// int32 tables), the calls into the CUDA library, and the way back to maps.
#include "host_api.hpp"
#include "count_bound.hpp"

#include <algorithm>
#include <functional>
#include <chrono>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string_view>
#include <thread>
#include <unordered_set>

namespace blance {

namespace {

const Strs kNoStrs;
inline const Strs& deref(const OptStrs& s) { return s ? *s : kNoStrs; }

[[noreturn]] void invalid(const std::string& msg) { throw BlanceError(BLANCE_ERR_INVALID_ARG, "blance: " + msg); }

// fmt.Sprintf("%10d", v), plan.go:527,539
std::string pad10(long long v) {
  char buf[32];
  std::snprintf(buf, sizeof buf, "%10lld", v);
  return buf;
}

// strconv.Atoi (plan.go:525): optional sign, decimal digits, must fit int64.
bool go_atoi(const std::string& s, long long* out) {
  size_t i = 0;
  if (s.empty()) return false;
  bool neg = false;
  if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
  if (i >= s.size()) return false;
  unsigned long long acc = 0;
  const unsigned long long lim = neg ? (1ULL << 63) : (1ULL << 63) - 1;
  for (; i < s.size(); ++i) {
    if (s[i] < '0' || s[i] > '9') return false;
    unsigned d = unsigned(s[i] - '0');
    if (acc > (lim - d) / 10) return false;
    acc = acc * 10 + d;
  }
  *out = neg ? -(long long)acc : (long long)acc;
  return true;
}

// The name part of the partition sort key: the padded form first, the raw name as
// the final tie-break (plan.go:519-528, 512).
struct NameKey { std::string padded, raw; };
bool name_key_less(const NameKey& a, const NameKey& b) {
  if (a.padded != b.padded) return a.padded < b.padded;
  return a.raw < b.raw;
}

struct Interner {
  std::unordered_map<std::string, int32_t> ids;
  Strs names;
  int32_t get(const std::string& s) {
    auto it = ids.find(s);
    if (it != ids.end()) return it->second;
    int32_t id = int32_t(names.size());
    ids.emplace(s, id);
    names.push_back(s);
    return id;
  }
  int32_t find(const std::string& s) const {
    auto it = ids.find(s);
    return it == ids.end() ? -1 : it->second;
  }
};

// string_view -> dense index, open addressing; the views point into the caller's maps, which
// outlive the call.  Built single-threaded, read from many threads.
struct SvTable {
  std::vector<uint32_t> slots;                  // index + 1, 0 = empty
  std::vector<uint64_t> hashes;
  std::vector<std::string_view> keys;
  uint64_t mask = 0;
  static uint64_t hash(std::string_view s) {    // FNV-1a with a final mix
    uint64_t h = 1469598103934665603ull;
    for (unsigned char c : s) { h ^= c; h *= 1099511628211ull; }
    h ^= h >> 32; h *= 0x9E3779B97F4A7C15ull; h ^= h >> 29;
    return h;
  }
  void init(size_t n) {
    size_t cap = 16;
    while (cap < n * 2 + 2) cap <<= 1;
    slots.assign(cap, 0u);
    mask = cap - 1;
    hashes.reserve(n);
    keys.reserve(n);
  }
  int32_t find(std::string_view s, uint64_t h) const {
    if (slots.empty()) return -1;
    for (uint64_t i = h & mask;; i = (i + 1) & mask) {
      const uint32_t e = slots[i];
      if (!e) return -1;
      if (hashes[e - 1] == h && keys[e - 1] == s) return int32_t(e - 1);
    }
  }
  int32_t insert(std::string_view s, uint64_t h) {   // the index of s, new or old
    for (uint64_t i = h & mask;; i = (i + 1) & mask) {
      const uint32_t e = slots[i];
      if (!e) {
        keys.push_back(s);
        hashes.push_back(h);
        slots[i] = uint32_t(keys.size());
        return int32_t(keys.size() - 1);
      }
      if (hashes[e - 1] == h && keys[e - 1] == s) return int32_t(e - 1);
    }
  }
};

// ---- a little data parallelism for the million-partition maps (the per-partition work is independent) ----
std::atomic<int> g_host_threads{0};             // SetHostThreads; 0 = default

int max_threads() {
  const int forced = g_host_threads.load(std::memory_order_relaxed);
  if (forced >= 1) return forced;
  static const int n = [] {
    if (const char* e = std::getenv("BLANCE_HOST_THREADS")) { const int v = std::atoi(e); if (v >= 1) return std::min(v, 64); }
    const unsigned hc = std::thread::hardware_concurrency();
    return int(std::min(16u, std::max(1u, hc)));
  }();
  return n;
}

// f(begin, end, thread index); runs inline below 32 768 items
template <class F>
void parallel_for(size_t n, F f) {
  const int T = max_threads();
  if (T <= 1 || n < 32768) { if (n) f(size_t(0), n, 0); return; }
  std::vector<std::thread> th;
  const size_t chunk = (n + size_t(T) - 1) / size_t(T);
  for (int t = 1; t < T; ++t) {
    const size_t lo = std::min(n, chunk * size_t(t)), hi = std::min(n, lo + chunk);
    if (lo < hi) th.emplace_back([=] { f(lo, hi, t); });
  }
  f(size_t(0), std::min(n, chunk), 0);
  for (auto& x : th) x.join();
}

// chunk sorts in parallel, then pairwise merges
template <class T, class Less>
void parallel_sort(std::vector<T>& v, Less less) {
  const int TN = max_threads();
  if (TN <= 1 || v.size() < 65536) { std::sort(v.begin(), v.end(), less); return; }
  int parts = 1;
  while (parts * 2 <= TN) parts *= 2;
  const size_t n = v.size();
  std::vector<size_t> cut(size_t(parts) + 1);
  for (int i = 0; i <= parts; ++i) cut[size_t(i)] = n * size_t(i) / size_t(parts);
  {
    std::vector<std::thread> th;
    for (int i = 1; i < parts; ++i) th.emplace_back([&, i] { std::sort(v.begin() + long(cut[size_t(i)]), v.begin() + long(cut[size_t(i) + 1]), less); });
    std::sort(v.begin(), v.begin() + long(cut[1]), less);
    for (auto& x : th) x.join();
  }
  for (int width = 1; width < parts; width *= 2) {
    std::vector<std::thread> th;
    for (int i = 0; i + width < parts; i += 2 * width) {
      const size_t lo = cut[size_t(i)], mid = cut[size_t(i + width)], hi = cut[size_t(std::min(parts, i + 2 * width))];
      th.emplace_back([&, lo, mid, hi] { std::inplace_merge(v.begin() + long(lo), v.begin() + long(mid), v.begin() + long(hi), less); });
    }
    for (auto& x : th) x.join();
  }
}

// first error raised inside a parallel region
struct ErrorSlot {
  std::mutex mu;
  bool has = false;
  std::string msg;
  void set(const std::string& m) { std::lock_guard<std::mutex> g(mu); if (!has) { has = true; msg = m; } }
  void rethrow() { if (has) invalid(msg); }
};

// sortStateNames (plan.go:437-474).  Go starts from random map order and its
// comparator is inconsistent when name order disagrees with priority order (the
// reference is then non-deterministic); starting from ascending names and running
// Go's small-slice insertion sort gives (priority, name) order whenever the
// reference is deterministic.
// topPriorityStateName (plan.go:126-132): the state of minimum priority.  The reference walks the model in map order,
// so ties are random there; here the first in ascending name order wins.  "" for an empty model.
std::string top_priority_state_name(const PartitionModel& model) {
  Strs by_name;
  for (const auto& kv : model) by_name.push_back(kv.first);
  std::sort(by_name.begin(), by_name.end());
  std::string top;
  for (const auto& n : by_name)
    if (top.empty() || model.at(n).Priority < model.at(top).Priority) top = n;
  return top;
}

Strs sort_state_names(const PartitionModel& model) {
  Strs s;
  for (const auto& kv : model) s.push_back(kv.first);
  std::sort(s.begin(), s.end());
  auto less = [&](const std::string& i, const std::string& j) {
    return model.at(i).Priority < model.at(j).Priority || i < j;
  };
  for (size_t i = 1; i < s.size(); ++i)
    for (size_t j = i; j > 0 && less(s[j], s[j - 1]); --j) std::swap(s[j], s[j - 1]);
  return s;
}

// --- hierarchy as strings (plan.go:703-774), evaluated once per (rule, anchor) ---
struct Hierarchy {
  const std::unordered_map<std::string, std::string>* parents;
  std::unordered_map<std::string, Strs> children;
  std::unordered_map<std::string, Strs> leaves_cache;

  explicit Hierarchy(const std::unordered_map<std::string, std::string>* p) : parents(p) {
    Strs nodes;                                          // plan.go:705-716
    if (p) for (const auto& kv : *p) nodes.push_back(kv.first);
    std::sort(nodes.begin(), nodes.end());
    for (const auto& c : nodes) children[p->at(c)].push_back(c);
  }
  std::string ancestor(std::string node, int level) const {   // plan.go:755-762
    while (level > 0) {
      if (!parents) { node.clear(); }
      else { auto it = parents->find(node); node = it == parents->end() ? std::string() : it->second; }
      --level;
    }
    return node;
  }
  const Strs& leaves(const std::string& node, int depth = 0) {   // plan.go:764-774
    auto hit = leaves_cache.find(node);
    if (hit != leaves_cache.end()) return hit->second;
    if (depth > 4096) invalid("NodeHierarchy contains a cycle (the reference recurses forever)");
    Strs rv;
    auto it = children.find(node);
    if (it == children.end() || it->second.empty()) rv.push_back(node);
    else for (const auto& c : it->second) { const Strs& sub = leaves(c, depth + 1); rv.insert(rv.end(), sub.begin(), sub.end()); }
    return leaves_cache.emplace(node, std::move(rv)).first->second;
  }
};

[[noreturn]] void counts_too_large() { throw BlanceError(BLANCE_ERR_UNSUPPORTED, std::string("blance: ") + BLANCE_COUNT_BOUND_MSG); }

// a count of non-model states: beyond int32 the count bound (count_bound.hpp) fails as well
int32_t count_i32(long long v) {
  if (v < INT32_MIN || v > INT32_MAX) counts_too_large();
  return int32_t(v);
}

// The hierarchy bit sets of blance_plan_in (plan.go:174-226, 703-774): rule_off over the states of `state_names`,
// and ie_mask[r][a] for every node id a of `node_names` plus the "" anchor.  `ids` maps node_names to their ids;
// the first N are nodesAll.
void hierarchy_tables(const Strs& state_names, const Strs& node_names, const std::unordered_map<std::string, int32_t>& ids,
                      int32_t N, const std::optional<HierarchyRules>& rules_opt,
                      const std::optional<std::unordered_map<std::string, std::string>>& parents, std::vector<int32_t>* rule_off,
                      std::vector<uint32_t>* ie_mask, int32_t* n_rules, int32_t* n_hier_bits) {
  const int32_t S = int32_t(state_names.size()), NU = int32_t(node_names.size());
  rule_off->assign(size_t(S) + 1, 0);
  ie_mask->clear();
  *n_rules = 0;
  *n_hier_bits = N;
  if (!rules_opt) return;
  std::vector<HierarchyRule> rules;
  for (int32_t s = 0; s < S; ++s) {
    auto it = rules_opt->find(state_names[size_t(s)]);
    if (it != rules_opt->end())
      for (const auto& r : it->second) rules.push_back(r);
    (*rule_off)[size_t(s) + 1] = int32_t(rules.size());
  }
  *n_rules = int32_t(rules.size());
  if (*n_rules == 0) return;
  Hierarchy h(parents ? &*parents : nullptr);
  // pass 1: the lists, and the leaf names outside nodesAll
  Interner extra_bits;
  std::vector<std::vector<int32_t>> lists(size_t(*n_rules) * size_t(NU + 1));
  for (int32_t r = 0; r < *n_rules; ++r)
    for (int32_t a = 0; a <= NU; ++a) {
      const std::string anchor = a < NU ? node_names[size_t(a)] : std::string();
      const Strs& inc = h.leaves(h.ancestor(anchor, rules[size_t(r)].IncludeLevel));
      const Strs& exc = h.leaves(h.ancestor(anchor, rules[size_t(r)].ExcludeLevel));
      std::unordered_set<std::string> ex(exc.begin(), exc.end());
      auto& out = lists[size_t(r) * size_t(NU + 1) + size_t(a)];
      for (const auto& leaf : inc) {
        if (ex.count(leaf)) continue;                          // plan.go:733
        auto id = ids.find(leaf);
        if (id != ids.end() && id->second < N) out.push_back(id->second);
        else out.push_back(N + extra_bits.get(leaf));
      }
    }
  *n_hier_bits = N + int32_t(extra_bits.names.size());
  const size_t HW = size_t((*n_hier_bits + 31) / 32);
  ie_mask->assign(size_t(*n_rules) * size_t(NU + 1) * HW, 0u);
  for (size_t i = 0; i < lists.size(); ++i)
    for (int32_t b : lists[i]) (*ie_mask)[i * HW + size_t(b >> 5)] |= 1u << (b & 31);
}

// plan.go:544-545 dereferences prevMap[name] whenever nodesToRemove is non-empty
void check_remove_needs_prev(const InternedPlan& ip, const OptStrs& nodesToRemove, const std::string& who) {
  if (deref(nodesToRemove).empty()) return;
  for (size_t p = 0; p < ip.part_in_assign.size(); ++p)
    if (ip.part_in_assign[p] && !ip.part_in_prev[p])
      invalid(who + "partition '" + ip.part_names[p] + "' is being assigned with nodesToRemove set but is missing from prevMap (the reference panics, plan.go:544)");
}

}  // namespace

// ------------------------------------------------------------------------------------

// InternPlan, with each state's slot range at least min_width[state name] wide (when given): the shared layout of a
// scenario sweep whose scenarios raise constraints.
static std::unique_ptr<InternedPlan> intern_plan(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                                 const Strs& nodesAll, const OptStrs& nodesToRemove,
                                                 const OptStrs& nodesToAdd, const PartitionModel& model,
                                                 const PlanNextMapOptions& options,
                                                 const std::unordered_map<std::string, int>* min_width) {
  auto ip = std::make_unique<InternedPlan>();
  blance_plan_in& in = ip->in;

  // ---- nodes
  Interner nodes;
  for (const auto& n : nodesAll) {
    if (nodes.find(n) >= 0) invalid("nodesAll contains '" + n + "' twice");
    nodes.get(n);
  }
  const int32_t N = int32_t(nodesAll.size());
  SvTable node_tab;                              // read-only view of nodesAll for the parallel passes
  node_tab.init(size_t(N));
  for (const auto& n : nodesAll) node_tab.insert(n, SvTable::hash(n));

  // ---- states
  ip->state_names = sort_state_names(model);
  const int32_t S = int32_t(ip->state_names.size());
  std::unordered_map<std::string, int32_t> state_id;
  for (int32_t s = 0; s < S; ++s) state_id[ip->state_names[size_t(s)]] = s;
  ip->state_priority.resize(size_t(S));
  ip->state_constraints.resize(size_t(S));
  ip->state_stickiness.assign(size_t(S), 0);
  ip->state_has_stickiness.assign(size_t(S), 0);
  int32_t top_state = -1;
  for (int32_t s = 0; s < S; ++s) {
    const auto& name = ip->state_names[size_t(s)];
    const auto& ms = model.at(name);
    ip->state_priority[size_t(s)] = ms.Priority;
    int k = ms.Constraints;                                        // plan.go:308-319
    if (options.ModelStateConstraints) {
      auto it = options.ModelStateConstraints->find(name);
      if (it != options.ModelStateConstraints->end()) k = it->second;
    }
    ip->state_constraints[size_t(s)] = k;
    if (options.StateStickiness) {
      auto it = options.StateStickiness->find(name);
      if (it != options.StateStickiness->end()) { ip->state_stickiness[size_t(s)] = it->second; ip->state_has_stickiness[size_t(s)] = 1; }
    }
  }
  if (S > 0) top_state = state_id[top_priority_state_name(model)];
  // the model has a handful of states: comparing names beats hashing them
  auto find_state = [&](const std::string& name) -> int32_t {
    for (int32_t s = 0; s < S; ++s)
      if (ip->state_names[size_t(s)].size() == name.size() && ip->state_names[size_t(s)] == name) return s;
    return -1;
  };

  // ---- partitions, indexed in the name order of the partition sort key (plan.go:519-528, 512).
  // The maps are walked once into pointer arrays; everything per partition after that runs in parallel.
  using Entry = const PartitionMap::value_type*;
  const bool same_map = &prevMap == &partitionsToAssign;
  std::vector<Entry> pv, av;
  auto walk = [&](const PartitionMap& m, std::vector<Entry>& out) {     // bucket ranges in parallel
    out.resize(m.size());
    const size_t B = m.bucket_count();
    const int T = max_threads();
    if (T <= 1 || m.size() < 32768) { size_t i = 0; for (const auto& kv : m) out[i++] = &kv; return; }
    std::vector<std::vector<Entry>> part{size_t(T)};
    parallel_for(B, [&](size_t lo, size_t hi, int t) {
      auto& mine = part[size_t(t)];
      mine.reserve((hi - lo) * m.size() / B + 16);
      for (size_t b = lo; b < hi; ++b)
        for (auto it = m.begin(b); it != m.end(b); ++it) mine.push_back(&*it);
    });
    size_t i = 0;
    for (const auto& v : part) { std::copy(v.begin(), v.end(), out.begin() + long(i)); i += v.size(); }
  };
  walk(prevMap, pv);
  if (!same_map) walk(partitionsToAssign, av);
  auto check_names = [&](const std::vector<Entry>& v) {
    ErrorSlot err;
    parallel_for(v.size(), [&](size_t lo, size_t hi, int) {
      for (size_t i = lo; i < hi; ++i)
        if (!v[i]->second.Name.empty() && v[i]->second.Name != v[i]->first) {
          err.set("Partition.Name '" + v[i]->second.Name + "' differs from its map key '" + v[i]->first + "'");
          return;
        }
    });
    err.rethrow();
  };
  check_names(pv);
  check_names(av);
  // name -> unique index (u), in first-seen order: prevMap's entries, then the new ones of partitionsToAssign
  std::vector<uint64_t> hp(pv.size()), ha(av.size());
  parallel_for(pv.size(), [&](size_t lo, size_t hi, int) { for (size_t i = lo; i < hi; ++i) hp[i] = SvTable::hash(pv[i]->first); });
  parallel_for(av.size(), [&](size_t lo, size_t hi, int) { for (size_t i = lo; i < hi; ++i) ha[i] = SvTable::hash(av[i]->first); });
  SvTable names;
  names.init(pv.size() + av.size());
  for (size_t i = 0; i < pv.size(); ++i) names.insert(pv[i]->first, hp[i]);        // map keys are unique: u == i
  std::vector<int32_t> au(av.size());
  for (size_t i = 0; i < av.size(); ++i) au[i] = names.insert(av[i]->first, ha[i]);
  const size_t U = names.keys.size();
  const int32_t PU = int32_t(U);
  // sort keys: names that are small non-negative integers compare as integers ("%10d" of v < 10^10 is ten
  // characters wide, so the padded strings order like the numbers); anything else compares as the strings do
  struct SortKey { long long v; uint32_t u; uint32_t numeric; };
  std::vector<SortKey> keys(U);
  parallel_for(U, [&](size_t lo, size_t hi, int) {
    for (size_t i = lo; i < hi; ++i) {
      long long v = 0;
      const std::string raw(names.keys[i]);
      const bool num = go_atoi(raw, &v) && v >= 0 && v < 10000000000ll;
      keys[i] = SortKey{num ? v : 0, uint32_t(i), num ? 1u : 0u};
    }
  });
  auto padded_of = [&](const SortKey& k) -> std::string {
    std::string raw(names.keys[k.u]);
    if (k.numeric) return pad10(k.v);
    long long v;
    if (go_atoi(raw, &v) && v >= 0) return pad10(v);
    return raw;
  };
  auto key_less = [&](const SortKey& a, const SortKey& b) {
    if (a.numeric && b.numeric) {
      if (a.v != b.v) return a.v < b.v;
      return names.keys[a.u] < names.keys[b.u];
    }
    const std::string pa = padded_of(a), pb = padded_of(b);
    if (pa != pb) return pa < pb;
    return names.keys[a.u] < names.keys[b.u];
  };
  parallel_sort(keys, key_less);
  std::vector<int32_t> rank(U);                 // unique index -> partition id
  ip->part_names.resize(U);
  parallel_for(U, [&](size_t lo, size_t hi, int) {
    for (size_t p = lo; p < hi; ++p) { rank[keys[p].u] = int32_t(p); ip->part_names[p] = std::string(names.keys[keys[p].u]); }
  });
  auto part_of_prev = [&](size_t i) { return rank[i]; };
  auto part_of_assign = [&](size_t i) { return rank[size_t(au[i])]; };

  // ---- per-partition scalars
  ip->part_in_prev.assign(size_t(PU), 0);
  ip->part_in_assign.assign(size_t(PU), 0);
  ip->part_weight.assign(size_t(PU), 1);
  ip->part_has_weight.assign(size_t(PU), 0);
  ip->part_name_rank.resize(size_t(PU));
  for (int32_t p = 0; p < PU; ++p) ip->part_name_rank[size_t(p)] = p;
  if (options.PartitionWeights)
    for (const auto& kv : *options.PartitionWeights) {
      const int32_t u = names.find(kv.first, SvTable::hash(kv.first));
      if (u < 0) continue;
      ip->part_weight[size_t(rank[size_t(u)])] = kv.second;
      ip->part_has_weight[size_t(rank[size_t(u)])] = 1;
    }

  // ---- slot layout and rows.  A state's range holds max(constraints, longest input list).  The rows are
  // filled in ONE pass over the maps assuming the constraints are wide enough; a longer list (rare) only
  // records the width it needs and the pass is repeated with the right layout.
  std::vector<int32_t> cap(size_t(S), 0);
  for (int32_t s = 0; s < S; ++s) {
    cap[size_t(s)] = std::max(0, ip->state_constraints[size_t(s)]);
    if (min_width) {
      auto it = min_width->find(ip->state_names[size_t(s)]);
      if (it != min_width->end()) cap[size_t(s)] = std::max(cap[size_t(s)], it->second);
    }
  }
  struct Extra { int32_t part; int32_t node; };
  struct Unknown { size_t pos; int which; const std::string* name; };   // a row cell (or extras entry) naming a node outside nodesAll
  std::vector<Extra> extras;   // prevMap entries under non-model states (only feed tot)
  int32_t SL = 0;
  for (int attempt = 0;; ++attempt) {
    ip->state_slot_off.assign(size_t(S) + 1, 0);
    for (int32_t s = 0; s < S; ++s) ip->state_slot_off[size_t(s) + 1] = ip->state_slot_off[size_t(s)] + cap[size_t(s)];
    SL = ip->state_slot_off[size_t(S)];
    extras.clear();
    std::vector<int32_t> need = cap;
    auto fill = [&](const std::vector<Entry>& v, bool from_prev, std::vector<int32_t>& rows, std::vector<uint8_t>& shape,
                    std::vector<uint8_t>& present, bool is_prev, bool must_be_model) {
      const int T = max_threads();
      ErrorSlot err;
      std::vector<std::vector<Extra>> textra{size_t(T)};
      std::vector<std::vector<Unknown>> tunk{size_t(T)};
      std::vector<std::vector<int32_t>> tneed(size_t(T), std::vector<int32_t>(size_t(S), 0));
      parallel_for(v.size(), [&](size_t lo, size_t hi, int t) {
        for (size_t i = lo; i < hi; ++i) {
          const int32_t p = from_prev ? part_of_prev(i) : part_of_assign(i);
          present[size_t(p)] |= 1;
          for (const auto& sn : v[i]->second.NodesByState) {
            const int32_t s = find_state(sn.first);
            if (s < 0) {
              if (must_be_model) {
                err.set("partition '" + v[i]->first + "' has state '" + sn.first + "' that is not in the model (the reference panics, plan.go:148)");
                return;
              }
              if (is_prev) present[size_t(p)] = 3;        // a key outside the model: never DeepEqual (plan.go:38)
              if (is_prev)
                for (const auto& n : deref(sn.second)) {
                  const int32_t id = node_tab.find(n, SvTable::hash(n));
                  if (id < 0) tunk[size_t(t)].push_back({textra[size_t(t)].size(), -1, &n});
                  textra[size_t(t)].push_back({p, id});
                }
              continue;
            }
            shape[size_t(p) * size_t(S) + size_t(s)] = sn.second ? BLANCE_SHAPE_LIST : BLANCE_SHAPE_NIL;
            const Strs& list = deref(sn.second);
            if (int32_t(list.size()) > cap[size_t(s)]) { tneed[size_t(t)][size_t(s)] = std::max(tneed[size_t(t)][size_t(s)], int32_t(list.size())); continue; }
            size_t pos = size_t(p) * size_t(SL) + size_t(ip->state_slot_off[size_t(s)]);
            for (const auto& n : list) {
              const int32_t id = node_tab.find(n, SvTable::hash(n));
              if (id >= 0) rows[pos] = id;
              else tunk[size_t(t)].push_back({pos, 0, &n});
              ++pos;
            }
          }
        }
      });
      err.rethrow();
      // names outside nodesAll get their ids here, in a fixed order (thread, then position)
      for (int t = 0; t < T; ++t) {
        for (const auto& u : tunk[size_t(t)]) {
          const int32_t id = nodes.get(*u.name);
          if (u.which >= 0) rows[u.pos] = id;
          else textra[size_t(t)][u.pos].node = id;
        }
        extras.insert(extras.end(), textra[size_t(t)].begin(), textra[size_t(t)].end());
        for (int32_t s = 0; s < S; ++s) need[size_t(s)] = std::max(need[size_t(s)], tneed[size_t(t)][size_t(s)]);
      }
    };
    ip->prev_rows.assign(size_t(PU) * size_t(SL), BLANCE_NO_NODE);
    ip->prev_shape.assign(size_t(PU) * size_t(S), BLANCE_SHAPE_ABSENT);
    fill(pv, true, ip->prev_rows, ip->prev_shape, ip->part_in_prev, true, same_map);
    if (!same_map) {
      ip->cur_rows.assign(size_t(PU) * size_t(SL), BLANCE_NO_NODE);
      ip->cur_shape.assign(size_t(PU) * size_t(S), BLANCE_SHAPE_ABSENT);
      fill(av, false, ip->cur_rows, ip->cur_shape, ip->part_in_assign, false, true);
    }
    if (need == cap) break;
    if (attempt >= 1) invalid("internal: slot layout did not settle");
    cap = need;
  }
  if (same_map) {
    ip->cur_rows = ip->prev_rows;
    ip->cur_shape = ip->prev_shape;
    ip->part_in_assign = ip->part_in_prev;
  }

  // ---- node flags (after every name that can occur has been interned)
  for (const auto& n : deref(nodesToRemove)) nodes.get(n);
  for (const auto& n : deref(nodesToAdd)) nodes.get(n);
  const int32_t NU = int32_t(nodes.names.size());
  ip->node_removed.assign(size_t(NU), 0);
  ip->node_added.assign(size_t(NU), 0);
  for (const auto& n : deref(nodesToRemove)) ip->node_removed[size_t(nodes.find(n))] = 1;
  for (const auto& n : deref(nodesToAdd)) ip->node_added[size_t(nodes.find(n))] = 1;
  ip->node_weight.assign(size_t(N), 0);
  ip->node_has_weight.assign(size_t(N), 0);
  if (options.NodeWeights)
    for (const auto& kv : *options.NodeWeights) {
      int32_t id = nodes.find(kv.first);
      if (id < 0 || id >= N) continue;
      ip->node_weight[size_t(id)] = kv.second;
      ip->node_has_weight[size_t(id)] = 1;
    }

  check_remove_needs_prev(*ip, nodesToRemove, "");

  // ---- counts under non-model states
  ip->extra_tot_first.assign(size_t(N), 0);
  ip->extra_tot_rest.assign(size_t(N), 0);
  ip->extra_part.clear();
  ip->extra_node.clear();
  for (const auto& e : extras) {
    ip->extra_part.push_back(e.part);
    ip->extra_node.push_back(e.node);
    if (e.node >= N) continue;
    long long w = (options.PartitionWeights && ip->part_has_weight[size_t(e.part)]) ? ip->part_weight[size_t(e.part)] : 1;
    ip->extra_tot_first[size_t(e.node)] = count_i32((long long)ip->extra_tot_first[size_t(e.node)] + w);
    if (!ip->part_in_assign[size_t(e.part)])
      ip->extra_tot_rest[size_t(e.node)] = count_i32((long long)ip->extra_tot_rest[size_t(e.node)] + w);
  }

  // ---- hierarchy bit sets
  int32_t n_rules = 0, n_hier_bits = N;
  hierarchy_tables(ip->state_names, nodes.names, nodes.ids, N, options.HierarchyRules, options.NodeHierarchy, &ip->rule_off,
                   &ip->ie_mask, &n_rules, &n_hier_bits);

  ip->node_names = nodes.names;

  in.n_nodes = N; in.n_node_ids = NU; in.n_states = S; in.n_parts = PU; in.n_slots = SL;
  in.max_iters = options.MaxIterationsPerPlan;
  in.top_state = top_state < 0 ? 0 : top_state;
  in.booster_kind = options.NodeScoreBooster;
  in.add_is_nil = nodesToAdd ? 0 : 1;
  in.has_part_weights = options.PartitionWeights ? 1 : 0;
  in.has_node_weights = options.NodeWeights ? 1 : 0;
  in.has_hier_rules = options.HierarchyRules ? 1 : 0;
  in.state_priority = ip->state_priority.data();
  in.state_constraints = ip->state_constraints.data();
  in.state_slot_off = ip->state_slot_off.data();
  in.state_stickiness = ip->state_stickiness.data();
  in.state_has_stickiness = ip->state_has_stickiness.data();
  in.node_removed = ip->node_removed.data();
  in.node_added = ip->node_added.data();
  in.node_weight = ip->node_weight.data();
  in.node_has_weight = ip->node_has_weight.data();
  in.part_in_prev = ip->part_in_prev.data();
  in.part_in_assign = ip->part_in_assign.data();
  in.part_weight = ip->part_weight.data();
  in.part_has_weight = ip->part_has_weight.data();
  in.part_name_rank = ip->part_name_rank.data();
  in.prev_rows = ip->prev_rows.data();
  in.prev_shape = ip->prev_shape.data();
  in.cur_rows = ip->cur_rows.data();
  in.cur_shape = ip->cur_shape.data();
  in.extra_tot_first = ip->extra_tot_first.data();
  in.extra_tot_rest = ip->extra_tot_rest.data();
  in.n_rules = n_rules;
  in.n_hier_bits = n_hier_bits;
  in.rule_off = ip->rule_off.data();
  in.ie_mask = ip->ie_mask.empty() ? nullptr : ip->ie_mask.data();
  in.engine = options.Engine;
  if (!count_bound_fits(in)) counts_too_large();
  return ip;
}

std::unique_ptr<InternedPlan> InternPlan(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                         const Strs& nodesAll, const OptStrs& nodesToRemove,
                                         const OptStrs& nodesToAdd, const PartitionModel& model,
                                         const PlanNextMapOptions& options) {
  return intern_plan(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, options, nullptr);
}

PlanOutBuffers::PlanOutBuffers(const InternedPlan& ip) {
  next_rows.assign(size_t(ip.in.n_parts) * size_t(ip.in.n_slots) + 1, BLANCE_NO_NODE);
  next_shape.assign(size_t(ip.in.n_parts) * size_t(ip.in.n_states) + 1, 0);
  warn.assign(size_t(ip.in.n_parts) * size_t(ip.in.n_states) + 1, 0);
  out.next_rows = next_rows.data();
  out.next_shape = next_shape.data();
  out.warn = warn.data();
}

static PartitionMap unintern_plan(const InternedPlan& ip, const PlanOutBuffers& ob, Warnings* warnings, const int32_t* constraints);

PartitionMap UninternPlan(const InternedPlan& ip, const PlanOutBuffers& ob, Warnings* warnings) {
  return unintern_plan(ip, ob, warnings, ip.state_constraints.data());
}

// UninternPlan whose warnings name `constraints` (a scenario's own) instead of the tables' constraints
static PartitionMap unintern_plan(const InternedPlan& ip, const PlanOutBuffers& ob, Warnings* warnings, const int32_t* constraints) {
  const blance_plan_in& in = ip.in;
  // the assigned partitions (plan.go:326-330), built in parallel, then moved into the map
  std::vector<int32_t> ids;
  ids.reserve(size_t(in.n_parts));
  for (int32_t p = 0; p < in.n_parts; ++p)
    if (ip.part_in_assign[size_t(p)]) ids.push_back(p);
  std::vector<Partition> parts(ids.size());
  parallel_for(ids.size(), [&](size_t lo, size_t hi, int) {
    for (size_t i = lo; i < hi; ++i) {
      const int32_t p = ids[i];
      Partition& part = parts[i];
      part.Name = ip.part_names[size_t(p)];
      const int32_t* row = ob.next_rows.data() + size_t(p) * size_t(in.n_slots);
      for (int32_t s = 0; s < in.n_states; ++s) {
        const uint8_t sh = ob.next_shape[size_t(p) * size_t(in.n_states) + size_t(s)];
        if (sh == BLANCE_SHAPE_ABSENT) continue;
        if (sh == BLANCE_SHAPE_NIL) { part.NodesByState[ip.state_names[size_t(s)]] = std::nullopt; continue; }
        Strs list;
        for (int32_t j = ip.state_slot_off[size_t(s)]; j < ip.state_slot_off[size_t(s) + 1] && row[j] != BLANCE_NO_NODE; ++j)
          list.push_back(ip.node_names[size_t(row[j])]);
        part.NodesByState[ip.state_names[size_t(s)]] = std::move(list);
      }
    }
  });
  PartitionMap next;
  next.reserve(ids.size());
  for (size_t i = 0; i < ids.size(); ++i) {
    const int32_t p = ids[i];
    if (warnings)
      for (int32_t s = 0; s < in.n_states; ++s)
        if (ob.warn[size_t(p) * size_t(in.n_states) + size_t(s)]) {
          char buf[32];                                              // plan.go:231-234
          std::snprintf(buf, sizeof buf, "%d", constraints[s]);
          (*warnings)[parts[i].Name].push_back(std::string("could not meet constraints: ") + buf +
                                               ", stateName: " + ip.state_names[size_t(s)] +
                                               ", partitionName: " + parts[i].Name);
        }
    std::string key = parts[i].Name;
    next.emplace(std::move(key), std::move(parts[i]));
  }
  return next;
}

// ---- the JSON wire form (api.go:30,35) --------------------------------------------------------------------
// encoding/json, default options: strings are quoted with ", \\ and control characters escaped (\n \r \t short
// forms, others \u00XX), <, > and & as \u003c \u003e \u0026 (HTML-safe), U+2028 / U+2029 as \u2028 / \u2029,
// invalid UTF-8 as U+FFFD; map keys are sorted by their bytes; a nil slice is null.
static void json_string(std::string& out, const std::string& v) {
  static const char* hex = "0123456789abcdef";
  out.push_back('"');
  const unsigned char* p = reinterpret_cast<const unsigned char*>(v.data());
  const size_t n = v.size();
  for (size_t i = 0; i < n;) {
    const unsigned char c = p[i];
    if (c < 0x80) {
      if (c == '"' || c == '\\') { out.push_back('\\'); out.push_back(char(c)); }
      else if (c == '\n') out += "\\n";
      else if (c == '\r') out += "\\r";
      else if (c == '\t') out += "\\t";
      else if (c < 0x20 || c == '<' || c == '>' || c == '&') { out += "\\u00"; out.push_back(hex[c >> 4]); out.push_back(hex[c & 15]); }
      else out.push_back(char(c));
      ++i;
      continue;
    }
    // decode one UTF-8 sequence the way Go's utf8.DecodeRuneInString does (shortest form, no surrogates, <= U+10FFFF)
    size_t len = 0;
    uint32_t cp = 0;
    if (c >= 0xC2 && c <= 0xDF) { len = 2; cp = c & 0x1F; }
    else if (c >= 0xE0 && c <= 0xEF) { len = 3; cp = c & 0x0F; }
    else if (c >= 0xF0 && c <= 0xF4) { len = 4; cp = c & 0x07; }
    bool ok = len != 0 && i + len <= n;
    for (size_t k = 1; ok && k < len; ++k) {
      const unsigned char d = p[i + k];
      unsigned char lo = 0x80, hi = 0xBF;
      if (k == 1) {
        if (c == 0xE0) lo = 0xA0;
        if (c == 0xED) hi = 0x9F;
        if (c == 0xF0) lo = 0x90;
        if (c == 0xF4) hi = 0x8F;
      }
      if (d < lo || d > hi) ok = false;
      cp = (cp << 6) | (d & 0x3F);
    }
    if (!ok) { out += "\\ufffd"; ++i; continue; }
    if (cp == 0x2028 || cp == 0x2029) { out += "\\u202"; out.push_back(hex[cp & 15]); }
    else out.append(v, i, len);
    i += len;
  }
  out.push_back('"');
}

template <class GetList>   // GetList(state index) -> (present, is_nil, list writer)
static void json_partition(std::string& out, const std::string& name, const std::vector<std::pair<const std::string*, const OptStrs*>>& states) {
  out += "{\"name\":";
  json_string(out, name);
  out += ",\"nodesByState\":{";
  bool first = true;
  for (const auto& st : states) {
    if (!first) out.push_back(',');
    first = false;
    json_string(out, *st.first);
    out.push_back(':');
    if (!*st.second) { out += "null"; continue; }
    out.push_back('[');
    bool f2 = true;
    for (const auto& n : **st.second) {
      if (!f2) out.push_back(',');
      f2 = false;
      json_string(out, n);
    }
    out.push_back(']');
  }
  out += "}}";
}

std::string PartitionMapToJSON(const PartitionMap& m) {
  std::vector<const std::pair<const std::string, Partition>*> entries;
  entries.reserve(m.size());
  for (const auto& kv : m) entries.push_back(&kv);
  std::sort(entries.begin(), entries.end(), [](auto* a, auto* b) { return a->first < b->first; });   // byte order = Go's key order
  std::vector<std::string> chunks(entries.size());
  parallel_for(entries.size(), [&](size_t lo, size_t hi, int) {
    std::vector<std::pair<const std::string*, const OptStrs*>> states;
    for (size_t i = lo; i < hi; ++i) {
      const Partition& part = entries[i]->second;
      states.clear();
      for (const auto& kv : part.NodesByState) states.push_back({&kv.first, &kv.second});
      std::sort(states.begin(), states.end(), [](const auto& a, const auto& b) { return *a.first < *b.first; });
      std::string& out = chunks[i];
      json_string(out, entries[i]->first);
      out.push_back(':');
      json_partition<int>(out, part.Name, states);
    }
  });
  size_t total = 2;
  for (const auto& c : chunks) total += c.size() + 1;
  std::string out;
  out.reserve(total);
  out.push_back('{');
  for (size_t i = 0; i < chunks.size(); ++i) {
    if (i) out.push_back(',');
    out += chunks[i];
  }
  out.push_back('}');
  return out;
}

// rows -> JSON directly (the next map of a plan; same bytes as PartitionMapToJSON(UninternPlan(...)))
std::string PlanResultToJSON(const InternedPlan& ip, const PlanOutBuffers& ob) {
  const blance_plan_in& in = ip.in;
  std::vector<int32_t> ids;
  for (int32_t p = 0; p < in.n_parts; ++p)
    if (ip.part_in_assign[size_t(p)]) ids.push_back(p);
  std::sort(ids.begin(), ids.end(), [&](int32_t a, int32_t b) { return ip.part_names[size_t(a)] < ip.part_names[size_t(b)]; });
  std::vector<int32_t> state_order(size_t(in.n_states));
  for (int32_t s = 0; s < in.n_states; ++s) state_order[size_t(s)] = s;
  std::sort(state_order.begin(), state_order.end(), [&](int32_t a, int32_t b) { return ip.state_names[size_t(a)] < ip.state_names[size_t(b)]; });
  std::vector<std::string> chunks(ids.size());
  parallel_for(ids.size(), [&](size_t lo, size_t hi, int) {
    std::vector<OptStrs> lists(size_t(in.n_states));
    std::vector<std::pair<const std::string*, const OptStrs*>> states;
    for (size_t i = lo; i < hi; ++i) {
      const int32_t p = ids[i];
      const int32_t* row = ob.next_rows.data() + size_t(p) * size_t(in.n_slots);
      states.clear();
      for (int32_t s : state_order) {
        const uint8_t sh = ob.next_shape[size_t(p) * size_t(in.n_states) + size_t(s)];
        if (sh == BLANCE_SHAPE_ABSENT) continue;
        OptStrs& l = lists[size_t(s)];
        if (sh == BLANCE_SHAPE_NIL) l = std::nullopt;
        else {
          l = Strs{};
          for (int32_t j = ip.state_slot_off[size_t(s)]; j < ip.state_slot_off[size_t(s) + 1] && row[j] != BLANCE_NO_NODE; ++j)
            l->push_back(ip.node_names[size_t(row[j])]);
        }
        states.push_back({&ip.state_names[size_t(s)], &l});
      }
      std::string& out = chunks[i];
      json_string(out, ip.part_names[size_t(p)]);
      out.push_back(':');
      json_partition<int>(out, ip.part_names[size_t(p)], states);
    }
  });
  std::string out;
  size_t total = 2;
  for (const auto& c : chunks) total += c.size() + 1;
  out.reserve(total);
  out.push_back('{');
  for (size_t i = 0; i < chunks.size(); ++i) {
    if (i) out.push_back(',');
    out += chunks[i];
  }
  out.push_back('}');
  return out;
}

// plan.go:49-52: after any non-matching iteration the caller's maps hold the new partitions; when the loop
// ends their content equals the returned map.  Map surgery (new keys) is serial, the deep copies are not.
void ReplayCallerMutation(const PartitionMap& next, PartitionMap& prevMap, PartitionMap& partitionsToAssign) {
  const bool same = &prevMap == &partitionsToAssign;
  std::vector<const Partition*> src;
  std::vector<Partition*> dst_prev, dst_assign;
  src.reserve(next.size());
  dst_prev.reserve(next.size());
  if (!same) dst_assign.reserve(next.size());
  for (const auto& kv : next) {
    src.push_back(&kv.second);
    dst_prev.push_back(&prevMap[kv.first]);
    if (!same) dst_assign.push_back(&partitionsToAssign[kv.first]);
  }
  parallel_for(src.size(), [&](size_t lo, size_t hi, int) {
    for (size_t i = lo; i < hi; ++i) {
      *dst_prev[i] = *src[i];
      if (!same) *dst_assign[i] = *src[i];
    }
  });
}

void SetHostThreads(int n) { g_host_threads.store(n < 0 ? 0 : (n > 64 ? 64 : n), std::memory_order_relaxed); }
int HostThreads() { return max_threads(); }

blance_ctx* DefaultContext() {
  static std::mutex mu;
  static blance_ctx* ctx = nullptr;
  std::lock_guard<std::mutex> g(mu);
  if (!ctx) {
    int st = blance_ctx_create(&ctx, -1);
    if (st != BLANCE_OK) {
      ctx = nullptr;
      throw BlanceError(st, std::string("blance_ctx_create failed: ") + blance_last_error(nullptr));
    }
  }
  return ctx;
}

PartitionMap PlanNextMapEx(PartitionMap& prevMap, PartitionMap& partitionsToAssign, const Strs& nodesAll,
                           const OptStrs& nodesToRemove, const OptStrs& nodesToAdd,
                           const PartitionModel& model, const PlanNextMapOptions& options,
                           Warnings* warnings, PlanStats* stats) {
  if (warnings) warnings->clear();
  using clk = std::chrono::steady_clock;
  auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  const auto t0 = clk::now();
  auto ip = InternPlan(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, options);
  PlanOutBuffers ob(*ip);
  const auto t1 = clk::now();
  blance_ctx* ctx = DefaultContext();
  int st = blance_plan_next_map(ctx, &ip->in, &ob.out);
  if (st != BLANCE_OK) throw BlanceError(st, std::string("blance_plan_next_map failed: ") + blance_last_error(ctx));
  const auto t2 = clk::now();
  if (stats) {
    stats->iters_run = ob.out.iters_run; stats->converged = ob.out.converged; stats->steps = ob.out.steps;
    stats->device_ms = ob.out.device_ms; stats->kernel_ms = ob.out.kernel_ms; stats->pass_ms = ob.out.pass_ms;
    stats->intern_ms = ms(t0, t1); stats->call_ms = ms(t1, t2);
  }
  if (ob.out.iters_run <= 0) return PartitionMap{};                  // MaxIterationsPerPlan <= 0: plan.go:32,57
  PartitionMap next = UninternPlan(*ip, ob, warnings);
  const auto t3 = clk::now();
  if (ob.out.iters_run >= 2 || !ob.out.converged) ReplayCallerMutation(next, prevMap, partitionsToAssign);
  if (stats) { stats->unintern_ms = ms(t2, t3); stats->mutate_ms = ms(t3, clk::now()); }
  return next;
}

// ------------------------------------------------------------------------------------
// What-if scenarios of one cluster

namespace {

constexpr int kMaxConstraints = 16;   // BL_K_MAX of the device (device_types.cuh)

// ModelStateConstraints of `state` in scenario `sc` (plan.go:308-319 on the substituted options)
int scenario_constraint(const PartitionModel& model, const PlanNextMapOptions& options, const Scenario& sc, const std::string& state) {
  int k = model.at(state).Constraints;
  const auto& msc = sc.ModelStateConstraints ? *sc.ModelStateConstraints : options.ModelStateConstraints;
  if (msc) {
    auto it = msc->find(state);
    if (it != msc->end()) k = it->second;
  }
  return k;
}

// The base tables of a scenario sweep.  The node-id space holds every name of every scenario's nodesToRemove and
// nodesToAdd (a removed name outside nodesAll still makes len(nodesToRemove) > 0, plan.go:543); the base's own node
// flags and weights are replaced per scenario.  Every state's slot range holds the largest constraint of any
// scenario: all scenarios share one row layout.
std::unique_ptr<InternedPlan> intern_scenario_base(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                                   const Strs& nodesAll, const PartitionModel& model,
                                                   const PlanNextMapOptions& options, const std::vector<Scenario>& scenarios) {
  Strs names;
  std::unordered_map<std::string, int> width;
  for (size_t i = 0; i < scenarios.size(); ++i) {
    const Scenario& sc = scenarios[i];
    for (const auto& n : deref(sc.NodesToRemove)) names.push_back(n);
    for (const auto& n : deref(sc.NodesToAdd)) names.push_back(n);
    if (!sc.ModelStateConstraints) continue;
    for (const auto& kv : model) {
      const int k = scenario_constraint(model, options, sc, kv.first);
      if (k > kMaxConstraints)
        throw BlanceError(BLANCE_ERR_UNSUPPORTED, "blance: scenario " + std::to_string(i) + ": constraints " + std::to_string(k) +
                                                      " of state '" + kv.first + "' are above 16, the device's limit");
      int& w = width[kv.first];
      w = std::max(w, k);
    }
  }
  return intern_plan(prevMap, partitionsToAssign, nodesAll, std::nullopt, OptStrs(std::move(names)), model, options, &width);
}

// One scenario's substitutions of the base tables: its node fields, and the option groups it sets
// (blance_scenario_opts; the arrays live here, scenario_opts() points at them).
struct ScenarioTables {
  std::vector<uint8_t> removed, added, has_weight;
  std::vector<int32_t> weight;
  int32_t add_is_nil = 0, has_node_weights = 0;
  uint32_t set = 0;
  std::vector<int32_t> constraints, stickiness;
  std::vector<uint8_t> has_stickiness;
  int32_t has_part_weights = 0;
  std::vector<int32_t> ow_part, ow_weight;          // weight overrides, ascending partition
  std::vector<uint8_t> ow_has;
  std::vector<int32_t> extra_first, extra_rest;     // empty: the base's
  int32_t has_hier_rules = 0, n_rules = 0, n_hier_bits = 0;
  std::vector<int32_t> rule_off;
  std::vector<uint32_t> ie_mask;
};

blance_scenario_opts scenario_opts(const ScenarioTables& t) {
  blance_scenario_opts o{};
  o.set = t.set;
  o.state_constraints = t.constraints.data();
  o.state_stickiness = t.stickiness.data();
  o.state_has_stickiness = t.has_stickiness.data();
  o.has_part_weights = t.has_part_weights;
  o.n_weight_overrides = int32_t(t.ow_part.size());
  o.ow_part = t.ow_part.data();
  o.ow_weight = t.ow_weight.data();
  o.ow_has = t.ow_has.data();
  o.extra_tot_first = t.extra_first.empty() ? nullptr : t.extra_first.data();
  o.extra_tot_rest = t.extra_rest.empty() ? nullptr : t.extra_rest.data();
  o.has_hier_rules = t.has_hier_rules;
  o.n_rules = t.n_rules;
  o.n_hier_bits = t.n_hier_bits;
  o.rule_off = t.rule_off.data();
  o.ie_mask = t.ie_mask.empty() ? nullptr : t.ie_mask.data();
  return o;
}

// partition name -> index of the base tables, built on first use (only scenarios with their own weights need it)
struct PartIndex {
  const InternedPlan& ip;
  std::unordered_map<std::string_view, int32_t> id;
  const std::unordered_map<std::string_view, int32_t>& get() {
    if (id.empty() && !ip.part_names.empty()) {
      id.reserve(ip.part_names.size());
      for (size_t p = 0; p < ip.part_names.size(); ++p) id.emplace(ip.part_names[p], int32_t(p));
    }
    return id;
  }
};

// who: "scenario i: " / "chain i, stage t: ".  check_prev: reject a removal with assigned partitions absent from
// prevMap (plan.go:544); a chain's later stages plan on a prevMap that holds every assigned partition.
ScenarioTables scenario_tables(const InternedPlan& ip, const PartitionModel& model, const Scenario& sc,
                               const PlanNextMapOptions& options, const std::string& who, PartIndex& parts, bool check_prev = true) {
  if (check_prev) check_remove_needs_prev(ip, sc.NodesToRemove, who);
  const int32_t N = ip.in.n_nodes, NU = ip.in.n_node_ids, S = ip.in.n_states;
  std::unordered_map<std::string, int32_t> id;
  id.reserve(size_t(NU));
  for (int32_t q = 0; q < NU; ++q) id.emplace(ip.node_names[size_t(q)], q);
  ScenarioTables t;
  t.removed.assign(size_t(NU) + 1, 0);
  t.added.assign(size_t(NU) + 1, 0);
  for (const auto& n : deref(sc.NodesToRemove)) t.removed[size_t(id.at(n))] = 1;
  for (const auto& n : deref(sc.NodesToAdd)) t.added[size_t(id.at(n))] = 1;
  t.add_is_nil = sc.NodesToAdd ? 0 : 1;
  const auto& weights = sc.NodeWeights ? *sc.NodeWeights : options.NodeWeights;
  t.weight.assign(size_t(N) + 1, 0);
  t.has_weight.assign(size_t(N) + 1, 0);
  t.has_node_weights = weights ? 1 : 0;
  if (weights)
    for (const auto& kv : *weights) {
      auto it = id.find(kv.first);
      if (it == id.end() || it->second >= N) continue;
      t.weight[size_t(it->second)] = kv.second;
      t.has_weight[size_t(it->second)] = 1;
    }

  if (sc.ModelStateConstraints) {
    t.set |= BLANCE_OPT_CONSTRAINTS;
    for (int32_t s = 0; s < S; ++s) t.constraints.push_back(scenario_constraint(model, options, sc, ip.state_names[size_t(s)]));
  }
  if (sc.StateStickiness) {
    t.set |= BLANCE_OPT_STICKINESS;
    t.stickiness.assign(size_t(S), 0);
    t.has_stickiness.assign(size_t(S), 0);
    if (*sc.StateStickiness)
      for (int32_t s = 0; s < S; ++s) {
        auto it = (*sc.StateStickiness)->find(ip.state_names[size_t(s)]);
        if (it != (*sc.StateStickiness)->end()) { t.stickiness[size_t(s)] = it->second; t.has_stickiness[size_t(s)] = 1; }
      }
  }
  if (sc.PartitionWeights) {
    t.set |= BLANCE_OPT_PART_WEIGHTS;
    const auto& pw = *sc.PartitionWeights;
    t.has_part_weights = pw ? 1 : 0;
    std::unordered_map<int32_t, int32_t> mine;      // the partitions of the maps this scenario weighs
    if (pw) {
      const auto& pid = parts.get();
      for (const auto& kv : *pw) {
        auto it = pid.find(kv.first);
        if (it == pid.end()) continue;                 // names outside the maps are ignored, as InternPlan does
        if (kv.second > 999999999)                     // the "%10d" rule of plan.go:539
          throw BlanceError(BLANCE_ERR_UNSUPPORTED, "blance: " + who + "partition weight of '" + kv.first + "' is above 999999999");
        mine.emplace(it->second, kv.second);
      }
      // overrides: partitions whose weight or presence differs from the base's (without weights the flags are unread)
      std::vector<std::pair<int32_t, int32_t>> diff;   // (partition, weight); presence below
      for (const auto& kv : mine)
        if (!ip.part_has_weight[size_t(kv.first)] || ip.part_weight[size_t(kv.first)] != kv.second) diff.emplace_back(kv.first, kv.second);
      for (int32_t p = 0; p < ip.in.n_parts; ++p)
        if (ip.part_has_weight[size_t(p)] && !mine.count(p)) diff.emplace_back(p, 1);
      std::sort(diff.begin(), diff.end());
      for (const auto& d : diff) {
        t.ow_part.push_back(d.first);
        t.ow_weight.push_back(d.second);
        t.ow_has.push_back(mine.count(d.first) ? 1 : 0);
      }
    }
    // extra_tot_* (host_api.cpp's counts of non-model states) only change when such a partition changes its weight
    auto w_base = [&](int32_t p) { return ip.in.has_part_weights && ip.part_has_weight[size_t(p)] ? ip.part_weight[size_t(p)] : 1; };
    auto w_mine = [&](int32_t p) {
      if (!pw) return 1;
      auto it = mine.find(p);
      return it == mine.end() ? 1 : it->second;
    };
    bool moved = false;
    for (int32_t p : ip.extra_part) moved |= w_base(p) != w_mine(p);
    if (moved) {
      t.extra_first.assign(size_t(N), 0);
      t.extra_rest.assign(size_t(N), 0);
      for (size_t e = 0; e < ip.extra_part.size(); ++e) {
        const int32_t p = ip.extra_part[e], q = ip.extra_node[e];
        if (q >= N) continue;
        t.extra_first[size_t(q)] = count_i32((long long)t.extra_first[size_t(q)] + w_mine(p));
        if (!ip.part_in_assign[size_t(p)]) t.extra_rest[size_t(q)] = count_i32((long long)t.extra_rest[size_t(q)] + w_mine(p));
      }
    }
  }
  if (sc.NodeHierarchy || sc.HierarchyRules) {
    t.set |= BLANCE_OPT_HIERARCHY;
    const auto& rules = sc.HierarchyRules ? *sc.HierarchyRules : options.HierarchyRules;
    const auto& parents = sc.NodeHierarchy ? *sc.NodeHierarchy : options.NodeHierarchy;
    t.has_hier_rules = rules ? 1 : 0;
    hierarchy_tables(ip.state_names, ip.node_names, id, N, rules, parents, &t.rule_off, &t.ie_mask, &t.n_rules, &t.n_hier_bits);
  }
  return t;
}

}  // namespace

// ------------------------------------------------------------------------------------
// The audit of a map, by name

namespace {

// The fault-domain forest of blance_audit_opts over interned node ids: the node names are vertices 0 .. NU-1, every other
// name of `parents` follows in byte order; a missing or "" parent is a root.
struct Forest {
  Strs names;                          // [V]
  std::vector<int32_t> parent;         // [V]; empty = nodes only
  blance_audit_opts opts{};
};

void build_forest(const Strs& node_names, const std::optional<std::unordered_map<std::string, std::string>>& parents, bool n2n, Forest* f) {
  f->names = node_names;
  f->opts = blance_audit_opts{};
  f->opts.flags = n2n ? BLANCE_AUDIT_N2N : 0;
  if (!parents) return;
  std::unordered_map<std::string, int32_t> id;
  for (size_t i = 0; i < f->names.size(); ++i) id.emplace(f->names[i], int32_t(i));
  Strs others;
  for (const auto& kv : *parents) { others.push_back(kv.first); others.push_back(kv.second); }
  std::sort(others.begin(), others.end());
  for (const auto& n : others)
    if (!n.empty() && id.emplace(n, int32_t(f->names.size())).second) f->names.push_back(n);
  f->parent.assign(f->names.size(), -1);
  for (const auto& kv : *parents)
    if (!kv.first.empty() && !kv.second.empty()) f->parent[size_t(id[kv.first])] = id[kv.second];
  f->opts.n_domains = int32_t(f->names.size() - node_names.size());
  f->opts.domain_parent = f->parent.data();
}

// Output buffers of one blance_audit_out over V vertices, R rules.
struct AuditBuffers {
  std::vector<int64_t> state, rule, dom;
  std::vector<int32_t> n2n;
  std::vector<uint8_t> flags;
  blance_audit_out out{};
  AuditBuffers(const InternedPlan& ip, size_t V, size_t R, bool want_n2n)
      : state(2 * size_t(ip.in.n_states) + 1), rule(2 * R + 1), dom(3 * V + 1),
        n2n(want_n2n ? size_t(ip.in.n_nodes) * size_t(ip.in.n_nodes) + 1 : 0), flags(size_t(ip.in.n_parts) + 1) {
    const size_t S = size_t(ip.in.n_states);
    out.short_slots = state.data(); out.over_slots = state.data() + S;
    out.rule_miss = rule.data(); out.rule_tested = rule.data() + R;
    out.dom_top = dom.data(); out.dom_all = dom.data() + V; out.dom_copies = dom.data() + 2 * V;
    out.n2n = want_n2n ? n2n.data() : nullptr;
    out.part_flags = flags.data();
  }
};

MapAudit name_audit(const InternedPlan& ip, const Forest& f, const int32_t* rule_off, const AuditBuffers& b, bool want_n2n) {
  MapAudit a;
  const blance_audit_out& o = b.out;
  const size_t S = size_t(ip.in.n_states), V = f.names.size(), N = size_t(ip.in.n_nodes);
  for (size_t s = 0; s < S; ++s) {
    if (o.short_slots[s]) a.ShortSlots[ip.state_names[s]] = o.short_slots[s];
    if (o.over_slots[s]) a.OverSlots[ip.state_names[s]] = o.over_slots[s];
    if (rule_off && rule_off[s + 1] > rule_off[s]) {
      a.RuleMiss[ip.state_names[s]].assign(o.rule_miss + rule_off[s], o.rule_miss + rule_off[s + 1]);
      a.RuleTested[ip.state_names[s]].assign(o.rule_tested + rule_off[s], o.rule_tested + rule_off[s + 1]);
    }
  }
  for (size_t v = 0; v < V; ++v) {
    if (o.dom_top[v]) a.DomTop[f.names[v]] = o.dom_top[v];
    if (o.dom_all[v]) a.DomAll[f.names[v]] = o.dom_all[v];
    if (o.dom_copies[v]) a.DomCopies[f.names[v]] = o.dom_copies[v];
  }
  a.ShortParts = o.short_parts; a.RuleMissParts = o.rule_miss_parts; a.NoTopParts = o.no_top_parts;
  for (size_t p = 0; p < size_t(ip.in.n_parts); ++p)
    if (o.part_flags[p]) a.PartFlags[ip.part_names[p]] = o.part_flags[p];
  a.HasFailoverSpread = want_n2n;
  if (want_n2n) {
    for (size_t x = 0; x < N; ++x)
      for (size_t y = 0; y < N; ++y)
        if (o.n2n[x * N + y]) a.FailoverSpread[ip.node_names[x]][ip.node_names[y]] = o.n2n[x * N + y];
    a.FailoverMax = std::max(0, o.n2n_max);
    if (o.n2n_max_a >= 0) { a.FailoverMaxFrom = ip.node_names[size_t(o.n2n_max_a)]; a.FailoverMaxTo = ip.node_names[size_t(o.n2n_max_b)]; }
  }
  return a;
}

}  // namespace

void AuditForest(const InternedPlan& ip, const std::optional<std::unordered_map<std::string, std::string>>& nodeHierarchy,
                 Strs* names, std::vector<int32_t>* parent) {
  Forest f;
  build_forest(ip.node_names, nodeHierarchy, false, &f);
  *names = std::move(f.names);
  *parent = std::move(f.parent);
}

MapAudit AuditMap(const PartitionMap& map, const Strs& nodesAll, const PartitionModel& model,
                  const PlanNextMapOptions& options, bool failoverSpread) {
  // the map interned as a prevMap with nothing to assign: each state's slot range holds its longest list, and state
  // names outside the model are allowed there (they are no copies)
  PlanNextMapOptions o;
  o.ModelStateConstraints = options.ModelStateConstraints;
  o.NodeHierarchy = options.NodeHierarchy;
  o.HierarchyRules = options.HierarchyRules;
  auto ip = InternPlan(map, PartitionMap{}, nodesAll, std::nullopt, std::nullopt, model, o);
  Forest f;
  build_forest(ip->node_names, options.NodeHierarchy, failoverSpread, &f);
  const size_t R = ip->in.has_hier_rules ? size_t(ip->in.n_rules) : 0;
  AuditBuffers b(*ip, f.names.size(), R, failoverSpread);
  blance_ctx* ctx = DefaultContext();
  const int st = blance_map_audit(ctx, &ip->in, ip->prev_rows.data(), ip->prev_shape.data(), &f.opts, &b.out);
  if (st != BLANCE_OK) throw BlanceError(st, std::string("blance_map_audit failed: ") + blance_last_error(ctx));
  return name_audit(*ip, f, ip->in.has_hier_rules ? ip->rule_off.data() : nullptr, b, failoverSpread);
}

std::unique_ptr<InternedPlan> InternScenario(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                             const Strs& nodesAll, const PartitionModel& model,
                                             const PlanNextMapOptions& options, const std::vector<Scenario>& scenarios,
                                             size_t index) {
  if (index >= scenarios.size()) invalid("InternScenario: scenario index out of range");
  auto ip = intern_scenario_base(prevMap, partitionsToAssign, nodesAll, model, options, scenarios);
  PartIndex parts{*ip, {}};
  ScenarioTables t = scenario_tables(*ip, model, scenarios[index], options, "scenario " + std::to_string(index) + ": ", parts);
  ip->node_removed = std::move(t.removed);
  ip->node_added = std::move(t.added);
  ip->node_weight = std::move(t.weight);
  ip->node_has_weight = std::move(t.has_weight);
  blance_plan_in& in = ip->in;
  in.add_is_nil = t.add_is_nil;
  in.has_node_weights = t.has_node_weights;
  if (t.set & BLANCE_OPT_CONSTRAINTS) ip->state_constraints = t.constraints;
  if (t.set & BLANCE_OPT_STICKINESS) { ip->state_stickiness = t.stickiness; ip->state_has_stickiness = t.has_stickiness; }
  if (t.set & BLANCE_OPT_PART_WEIGHTS) {
    in.has_part_weights = t.has_part_weights;
    for (size_t j = 0; j < t.ow_part.size(); ++j) {
      ip->part_weight[size_t(t.ow_part[j])] = t.ow_weight[j];
      ip->part_has_weight[size_t(t.ow_part[j])] = t.ow_has[j];
    }
    if (!t.extra_first.empty()) { ip->extra_tot_first = t.extra_first; ip->extra_tot_rest = t.extra_rest; }
  }
  if (t.set & BLANCE_OPT_HIERARCHY) {
    ip->rule_off = t.rule_off;
    ip->ie_mask = t.ie_mask;
    in.has_hier_rules = t.has_hier_rules; in.n_rules = t.n_rules; in.n_hier_bits = t.n_hier_bits;
  }
  in.node_removed = ip->node_removed.data();
  in.node_added = ip->node_added.data();
  in.node_weight = ip->node_weight.data();
  in.node_has_weight = ip->node_has_weight.data();
  in.state_constraints = ip->state_constraints.data();
  in.state_stickiness = ip->state_stickiness.data();
  in.state_has_stickiness = ip->state_has_stickiness.data();
  in.part_weight = ip->part_weight.data();
  in.part_has_weight = ip->part_has_weight.data();
  in.extra_tot_first = ip->extra_tot_first.data();
  in.extra_tot_rest = ip->extra_tot_rest.data();
  in.rule_off = ip->rule_off.data();
  in.ie_mask = ip->ie_mask.empty() ? nullptr : ip->ie_mask.data();
  return ip;
}

namespace {

const char* const kOpNames[] = {"add", "del", "promote", "demote"};   // enum blance_op_kind

// node_ops [NU][4] by node and op name, nonzero entries only
std::unordered_map<std::string, std::unordered_map<std::string, int64_t>> node_ops_by_name(const InternedPlan& ip, const int64_t* ops) {
  std::unordered_map<std::string, std::unordered_map<std::string, int64_t>> r;
  for (int32_t q = 0; q < ip.in.n_node_ids; ++q)
    for (int k = 0; k < 4; ++k)
      if (ops[size_t(q) * 4 + size_t(k)]) r[ip.node_names[size_t(q)]][kOpNames[k]] = ops[size_t(q) * 4 + size_t(k)];
  return r;
}

// One blance_scenario_out by name; `map` (rows copied out, or NULL) is uninterned under the constraints k.
ScenarioResult scenario_result(const InternedPlan& ip, const blance_scenario_out& o, const std::vector<int64_t>& ops,
                               const std::vector<int64_t>& load, PlanOutBuffers* map, const int32_t* k) {
  const int32_t NU = ip.in.n_node_ids, S = ip.in.n_states;
  ScenarioResult r;
  r.iters_run = o.iters_run; r.converged = o.converged; r.steps = o.steps; r.sticky_steps = o.sticky_steps;
  r.parts_moved = o.parts_moved; r.ops_total = o.ops_total; r.warn_parts = o.warn_parts;
  r.NodeOps = node_ops_by_name(ip, ops.data());
  for (int32_t s = 0; s < S; ++s)
    for (int32_t q = 0; q < NU; ++q)
      if (load[size_t(s) * size_t(NU) + size_t(q)])
        r.StateNodeLoad[ip.state_names[size_t(s)]][ip.node_names[size_t(q)]] = load[size_t(s) * size_t(NU) + size_t(q)];
  if (map) {
    r.HasMap = true;
    map->out.iters_run = o.iters_run;
    if (o.iters_run > 0) r.NextMap = unintern_plan(ip, *map, &r.NextWarnings, k);   // MaxIterationsPerPlan <= 0: plan.go:32,57
  }
  return r;
}

// Output buffers of one blance_exposure_out: series [BLANCE_EXPO_N][cap], V vertices, P partitions.
struct ExposureBuffers {
  std::vector<int64_t> series, dom_peak;
  std::vector<int32_t> dom_round, min_copies, no_top;
  std::vector<uint8_t> flags;
  blance_exposure_out out{};
  ExposureBuffers(size_t cap, size_t V, size_t P)
      : series(BLANCE_EXPO_N * cap + 1), dom_peak(V + 1), dom_round(V + 1), min_copies(P + 1), no_top(P + 1), flags(P + 1) {
    out.series = cap ? series.data() : nullptr; out.dom_peak = dom_peak.data(); out.dom_peak_round = dom_round.data();
    out.part_min_copies = min_copies.data(); out.part_no_top = no_top.data(); out.part_flags = flags.data();
  }
};

// One exposure by name: `cap` series values per metric were copied (the first min(R + 1, cap) are kept), vertices
// are vnames, partitions pnames.  Vertex- and partition-keyed fields keep positive entries only (a partition outside
// the exposed map reads -1 / 0 / 0 and is left out).
ExposureResult name_exposure(const ExposureBuffers& b, size_t cap, const Strs& vnames, const Strs& pnames) {
  static const char* kMetrics[BLANCE_EXPO_N] = {"NO_TOP", "MULTI_TOP", "SHORT", "ONE_COPY", "NO_COPY", "COPIES"};
  const blance_exposure_out& o = b.out;
  ExposureResult r;
  r.Rounds = o.rounds;
  r.KernelMs = o.kernel_ms;
  const size_t n = std::min(size_t(o.rounds) + 1, cap);
  for (size_t m = 0; m < BLANCE_EXPO_N; ++m) {
    r.Series[kMetrics[m]].assign(b.series.begin() + std::ptrdiff_t(m * cap), b.series.begin() + std::ptrdiff_t(m * cap + n));
    r.Peak[kMetrics[m]] = o.peak[m];
    r.PeakRound[kMetrics[m]] = o.peak_round[m];
    r.Area[kMetrics[m]] = o.area[m];
  }
  for (size_t v = 0; v < vnames.size(); ++v)
    if (b.dom_peak[v] > 0) { r.DomPeak[vnames[v]] = b.dom_peak[v]; r.DomPeakRound[vnames[v]] = b.dom_round[v]; }
  for (size_t p = 0; p < pnames.size(); ++p) {
    if (b.min_copies[p] > 0) r.PartMinCopies[pnames[p]] = b.min_copies[p];
    if (b.no_top[p] > 0) r.PartNoTop[pnames[p]] = b.no_top[p];
    if (b.flags[p]) r.PartFlags[pnames[p]] = b.flags[p];
  }
  return r;
}

// One schedule summary by name, at MaxConcurrentPartitionMovesPerNode `count`.
ScenarioSchedule name_schedule(const InternedPlan& ip, const blance_scenario_schedule_out& so, int count) {
  ScenarioSchedule s;
  s.MaxConcurrentPartitionMovesPerNode = count;
  s.Rounds = so.rounds; s.MovesDone = so.moves_done; s.StuckParts = so.stuck_parts; s.MaxBatch = so.max_batch;
  for (int32_t q = 0; q < ip.in.n_node_ids; ++q) {
    if (so.node_rounds[q]) s.NodeRounds[ip.node_names[size_t(q)]] = so.node_rounds[q];
    if (so.node_last_round[q]) s.NodeLastRound[ip.node_names[size_t(q)]] = so.node_last_round[q];
  }
  return s;
}

// Output buffers of n x nc blance_scenario_schedule_out (per-node arrays only, as ScenarioSchedule reports).
struct ScheduleBuffers {
  std::vector<blance_scenario_schedule_out> out;
  std::vector<int32_t> node_rounds, node_last;
  ScheduleBuffers(size_t count, size_t NU) : out(count), node_rounds(count * NU + 1), node_last(count * NU + 1) {
    for (size_t x = 0; x < count; ++x) {
      out[x] = blance_scenario_schedule_out{};
      out[x].node_rounds = node_rounds.data() + x * NU;
      out[x].node_last_round = node_last.data() + x * NU;
    }
  }
};

// Output buffers of one blance_chain_span_out: NU node ids, P partitions, V vertices; exposure arrays with `expo`.
struct SpanBuffers {
  std::vector<int32_t> node_rounds, min_copies, no_top, dom_stage, dom_round;
  std::vector<int64_t> node_last, part_done, dom_peak;
  std::vector<uint8_t> flags;
  blance_chain_span_out out{};
  SpanBuffers(size_t NU, size_t P, size_t V, bool expo)
      : node_rounds(NU + 1), min_copies(P + 1), no_top(P + 1), dom_stage(V + 1), dom_round(V + 1), node_last(NU + 1), part_done(P + 1),
        dom_peak(V + 1), flags(P + 1) {
    out.node_rounds = node_rounds.data(); out.node_last_round = node_last.data(); out.part_done_round = part_done.data();
    if (expo) {
      out.part_min_copies = min_copies.data(); out.part_no_top = no_top.data(); out.part_flags = flags.data();
      out.dom_peak = dom_peak.data(); out.dom_peak_stage = dom_stage.data(); out.dom_peak_round = dom_round.data();
    }
  }
};

ChainSpan name_span(const InternedPlan& ip, const SpanBuffers& b, int count, const Strs& vnames) {
  static const char* kMetrics[BLANCE_EXPO_N] = {"NO_TOP", "MULTI_TOP", "SHORT", "ONE_COPY", "NO_COPY", "COPIES"};
  const blance_chain_span_out& o = b.out;
  ChainSpan r;
  r.MaxConcurrentPartitionMovesPerNode = count;
  r.Rounds = o.rounds; r.MovesDone = o.moves_done; r.StuckParts = o.stuck_parts; r.MaxBatch = o.max_batch;
  for (int32_t q = 0; q < ip.in.n_node_ids; ++q) {
    if (b.node_rounds[size_t(q)]) r.NodeRounds[ip.node_names[size_t(q)]] = b.node_rounds[size_t(q)];
    if (b.node_last[size_t(q)]) r.NodeLastRound[ip.node_names[size_t(q)]] = b.node_last[size_t(q)];
  }
  const size_t P = ip.part_names.size();
  for (size_t p = 0; p < P; ++p)
    if (b.part_done[p]) r.PartDoneRound[ip.part_names[p]] = b.part_done[p];
  if (!o.part_min_copies) return r;
  for (size_t m = 0; m < BLANCE_EXPO_N; ++m) {
    r.Peak[kMetrics[m]] = o.peak[m]; r.Area[kMetrics[m]] = o.area[m];
    r.PeakStage[kMetrics[m]] = o.peak_stage[m]; r.PeakRound[kMetrics[m]] = o.peak_round[m];
  }
  for (size_t p = 0; p < P; ++p) {
    if (b.min_copies[p] > 0) r.PartMinCopies[ip.part_names[p]] = b.min_copies[p];
    if (b.no_top[p] > 0) r.PartNoTop[ip.part_names[p]] = b.no_top[p];
    if (b.flags[p]) r.PartFlags[ip.part_names[p]] = b.flags[p];
  }
  for (size_t v = 0; v < vnames.size(); ++v)
    if (b.dom_peak[v] > 0) {
      r.DomPeak[vnames[v]] = b.dom_peak[v]; r.DomPeakStage[vnames[v]] = b.dom_stage[v]; r.DomPeakRound[vnames[v]] = b.dom_round[v];
    }
  return r;
}

// The rule offsets and count a scenario audits with: its own when its options set the hierarchy, else the base's.
struct AuditRules {
  const int32_t* off = nullptr;
  int32_t n = 0;
};

AuditRules audit_rules(const ScenarioTables& t, const InternedPlan& ip) {
  if (t.set & BLANCE_OPT_HIERARCHY) return t.has_hier_rules ? AuditRules{t.rule_off.data(), t.n_rules} : AuditRules{};
  return ip.in.has_hier_rules ? AuditRules{ip.rule_off.data(), ip.in.n_rules} : AuditRules{};
}

// A blance_scenario_out into ops and load and, when the map is wanted, into map's rows, shape and warnings.
blance_scenario_out scenario_out(std::vector<int64_t>& ops, std::vector<int64_t>& load, PlanOutBuffers* map) {
  blance_scenario_out o{};
  o.node_ops = ops.data();
  o.state_node_load = load.data();
  if (map) {
    o.next_rows = map->next_rows.data();
    o.next_shape = map->next_shape.data();
    o.warn = map->warn.data();
  }
  return o;
}

// The schedule, audit and exposure outputs of n_out planned maps at nc counts each: schedules [n_out][nc], with audit
// audits [n_out] (map x audits with rules(x)), with exposure exposures [n_out][nc].  The exposures' forest is the
// options' NodeHierarchy, built also without exposure when `eforest_always` (a chain's spans are keyed by it).
struct AnalysisOutputs {
  const ScenarioAudit* audit;
  const bool exposure;
  const size_t cap;
  ScheduleBuffers sched;
  Forest forest, eforest;
  std::vector<std::unique_ptr<AuditBuffers>> abuf;
  std::vector<blance_audit_out> aout;
  std::vector<std::unique_ptr<ExposureBuffers>> ebuf;
  std::vector<blance_exposure_out> eout;
  template <class Rules>
  AnalysisOutputs(const InternedPlan& ip, const PlanNextMapOptions& options, size_t n_out, size_t nc, const ScenarioAudit* a,
                  const ScenarioExposure* e, bool eforest_always, Rules&& rules)
      : audit(a), exposure(e != nullptr), cap(e ? size_t(e->SeriesCap) : 0), sched(n_out * nc, size_t(ip.in.n_node_ids)) {
    if (audit) {
      build_forest(ip.node_names, options.NodeHierarchy, audit->FailoverSpread, &forest);
      for (size_t x = 0; x < n_out; ++x) {
        abuf.push_back(std::make_unique<AuditBuffers>(ip, forest.names.size(), size_t(rules(x).n), audit->FailoverSpread));
        aout.push_back(abuf.back()->out);
      }
    }
    if (exposure || eforest_always) build_forest(ip.node_names, options.NodeHierarchy, false, &eforest);
    for (size_t x = 0; exposure && x < n_out * nc; ++x) {
      ebuf.push_back(std::make_unique<ExposureBuffers>(cap, eforest.names.size(), size_t(ip.in.n_parts)));
      eout.push_back(ebuf.back()->out);
    }
  }
  // Map x's schedules at `counts`, audit (with the rule offsets rule_off) and exposures, into r.
  void name(const InternedPlan& ip, size_t x, const std::vector<int>& counts, const int32_t* rule_off, ScenarioResult& r) {
    const size_t nc = counts.size();
    for (size_t k = 0; k < nc; ++k) r.Schedules.push_back(name_schedule(ip, sched.out[x * nc + k], counts[k]));
    if (audit) {
      abuf[x]->out = aout[x];
      r.Audit = name_audit(ip, forest, rule_off, *abuf[x], audit->FailoverSpread);
    }
    for (size_t k = 0; exposure && k < nc; ++k) {
      ebuf[x * nc + k]->out = eout[x * nc + k];
      r.Exposures.push_back(name_exposure(*ebuf[x * nc + k], cap, eforest.names, ip.part_names));
    }
  }
};

}  // namespace

std::vector<ScenarioResult> PlanNextMapScenarios(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                                 const Strs& nodesAll, const PartitionModel& model,
                                                 const PlanNextMapOptions& options, const std::vector<Scenario>& scenarios,
                                                 bool favorMinNodes, const std::vector<int>& wantMaps, int maxConcurrent,
                                                 const std::vector<int>& scheduleConcurrency, const ScenarioAudit* audit,
                                                 const ScenarioExposure* exposure) {
  if (scenarios.empty()) invalid("PlanNextMapScenarios: no scenarios");
  if (exposure && scheduleConcurrency.empty()) invalid("PlanNextMapScenarios: an exposure needs scheduleConcurrency");
  if (exposure && exposure->SeriesCap < 0) invalid("PlanNextMapScenarios: SeriesCap is negative");
  auto ip = intern_scenario_base(prevMap, partitionsToAssign, nodesAll, model, options, scenarios);
  const size_t n = scenarios.size();
  PartIndex parts{*ip, {}};
  std::vector<ScenarioTables> tabs(n);
  for (size_t i = 0; i < n; ++i) tabs[i] = scenario_tables(*ip, model, scenarios[i], options, "scenario " + std::to_string(i) + ": ", parts);
  std::vector<bool> want(n, false);
  for (int i : wantMaps) {
    if (i < 0 || size_t(i) >= n) invalid("PlanNextMapScenarios: wantMaps index " + std::to_string(i) + " out of range");
    want[size_t(i)] = true;
  }
  const int32_t NU = ip->in.n_node_ids, S = ip->in.n_states;
  std::vector<blance_scenario> sc(n);
  std::vector<blance_scenario_opts> opts(n);
  std::vector<blance_scenario_out> out(n);
  std::vector<std::vector<int64_t>> ops(n, std::vector<int64_t>(size_t(NU) * 4 + 1)), load(n, std::vector<int64_t>(size_t(S) * size_t(NU) + 1));
  std::vector<std::unique_ptr<PlanOutBuffers>> maps(n);
  for (size_t i = 0; i < n; ++i) {
    sc[i] = blance_scenario{tabs[i].removed.data(), tabs[i].added.data(), tabs[i].add_is_nil, tabs[i].has_node_weights,
                            tabs[i].weight.data(), tabs[i].has_weight.data()};
    opts[i] = scenario_opts(tabs[i]);
    if (want[i]) maps[i] = std::make_unique<PlanOutBuffers>(*ip);
    out[i] = scenario_out(ops[i], load[i], maps[i].get());
  }
  const size_t nc = scheduleConcurrency.size();
  // the audits: one forest for all scenarios, each scenario's own rules
  AnalysisOutputs an(*ip, options, n, nc, audit, exposure, false, [&](size_t i) { return audit_rules(tabs[i], *ip); });
  blance_ctx* ctx = DefaultContext();
  const int st = exposure ? blance_plan_scenarios_exposure(ctx, &ip->in, int32_t(n), sc.data(), opts.data(), favorMinNodes ? 1 : 0, maxConcurrent,
                                                           int32_t(nc), scheduleConcurrency.data(), nullptr, out.data(), an.sched.out.data(),
                                                           audit ? &an.forest.opts : nullptr, audit ? an.aout.data() : nullptr, &an.eforest.opts,
                                                           int32_t(an.cap), an.eout.data())
                 : audit ? blance_plan_scenarios_audit(ctx, &ip->in, int32_t(n), sc.data(), opts.data(), favorMinNodes ? 1 : 0, maxConcurrent,
                                                     int32_t(nc), nc ? scheduleConcurrency.data() : nullptr, nullptr, out.data(),
                                                     nc ? an.sched.out.data() : nullptr, &an.forest.opts, an.aout.data())
                 : nc ? blance_plan_scenarios_schedule(ctx, &ip->in, int32_t(n), sc.data(), opts.data(), favorMinNodes ? 1 : 0, maxConcurrent,
                                                     int32_t(nc), scheduleConcurrency.data(), nullptr, out.data(), an.sched.out.data())
                    : blance_plan_scenarios_ex(ctx, &ip->in, int32_t(n), sc.data(), opts.data(), favorMinNodes ? 1 : 0, maxConcurrent,
                                               out.data());
  if (st != BLANCE_OK) throw BlanceError(st, std::string("blance_plan_scenarios failed: ") + blance_last_error(ctx));
  std::vector<ScenarioResult> res(n);
  for (size_t i = 0; i < n; ++i) {
    ScenarioResult& r = res[i];
    const int32_t* k = (tabs[i].set & BLANCE_OPT_CONSTRAINTS) ? tabs[i].constraints.data() : ip->state_constraints.data();
    r = scenario_result(*ip, out[i], ops[i], load[i], want[i] ? maps[i].get() : nullptr, k);
    an.name(*ip, i, scheduleConcurrency, audit_rules(tabs[i], *ip).off, r);
  }
  return res;
}

std::vector<ChainResult> PlanNextMapChains(const PartitionMap& prevMap, const PartitionMap& partitionsToAssign,
                                           const Strs& nodesAll, const PartitionModel& model,
                                           const PlanNextMapOptions& options, const std::vector<Chain>& chains,
                                           bool favorMinNodes, const std::vector<int>& wantMaps, int maxConcurrent,
                                           const std::vector<int>& scheduleConcurrency, const ScenarioAudit* audit,
                                           const ScenarioExposure* exposure, const std::vector<ChainBranch>* branches,
                                           std::vector<ChainResult>* branchResults) {
  if (chains.empty()) invalid("PlanNextMapChains: no chains");
  if ((audit || exposure) && scheduleConcurrency.empty()) invalid("PlanNextMapChains: an audit or exposure needs scheduleConcurrency");
  if (exposure && exposure->SeriesCap < 0) invalid("PlanNextMapChains: SeriesCap is negative");
  const size_t n = chains.size(), T = chains[0].Stages.size();
  if (T == 0) invalid("PlanNextMapChains: chain 0 has no stages");
  for (size_t i = 0; i < n; ++i)
    if (chains[i].Stages.size() != T)
      invalid("PlanNextMapChains: chain " + std::to_string(i) + " has " + std::to_string(chains[i].Stages.size()) +
              " stages, chain 0 has " + std::to_string(T) + " (chains of different lengths go in separate calls)");
  const size_t nb = branches ? branches->size() : 0, TB = nb ? (*branches)[0].Stages.size() : 0;
  if (nb && !branchResults) invalid("PlanNextMapChains: branches need branchResults");
  for (size_t b = 0; b < nb; ++b) {
    const ChainBranch& br = (*branches)[b];
    const std::string who = "PlanNextMapChains: branch " + std::to_string(b);
    if (br.Stages.size() != TB || TB == 0)
      invalid(who + " has " + std::to_string(br.Stages.size()) + " stages, branch 0 has " + std::to_string(TB) +
              " (every branch of one call has the same number of stages, at least one)");
    if (br.Chain < 0 || size_t(br.Chain) >= n) invalid(who + ": Chain outside [0, len(chains))");
    if (br.AfterStage < -1 || br.AfterStage >= int(T)) invalid(who + ": AfterStage outside [-1, stages)");
  }
  // every stage as a scenario: its node sets and weights, its chain's option fields and the stage's own; the trunk's
  // n x T stages first, then the branches' nb x TB
  auto stage_scenario = [](const Chain& ch, const ChainStage& cs, bool& own_opts) {
    Scenario sc = ch.Options;
    sc.NodesToRemove = cs.NodesToRemove;
    sc.NodesToAdd = cs.NodesToAdd;
    if (cs.NodeWeights) sc.NodeWeights = cs.NodeWeights;
    if (cs.ModelStateConstraints) sc.ModelStateConstraints = cs.ModelStateConstraints;
    if (cs.StateStickiness) sc.StateStickiness = cs.StateStickiness;
    if (cs.PartitionWeights) sc.PartitionWeights = cs.PartitionWeights;
    if (cs.NodeHierarchy) sc.NodeHierarchy = cs.NodeHierarchy;
    if (cs.HierarchyRules) sc.HierarchyRules = cs.HierarchyRules;
    own_opts |= cs.ModelStateConstraints || cs.StateStickiness || cs.PartitionWeights || cs.NodeHierarchy || cs.HierarchyRules;
    return sc;
  };
  const size_t NS = n * T + nb * TB;   // stages of the trunk and the branches
  std::vector<Scenario> flat(NS);
  bool stage_opts = nb > 0;            // some stage sets an option of its own (or branches): options per stage
  for (size_t i = 0; i < n; ++i)
    for (size_t t = 0; t < T; ++t) flat[i * T + t] = stage_scenario(chains[i], chains[i].Stages[t], stage_opts);
  for (size_t b = 0; b < nb; ++b)
    for (size_t u = 0; u < TB; ++u)
      flat[n * T + b * TB + u] = stage_scenario(chains[size_t((*branches)[b].Chain)], (*branches)[b].Stages[u], stage_opts);
  auto ip = intern_scenario_base(prevMap, partitionsToAssign, nodesAll, model, options, flat);
  const int32_t N = ip->in.n_nodes, NU = ip->in.n_node_ids, S = ip->in.n_states;
  std::unordered_map<std::string, int32_t> universe;
  for (int32_t q = 0; q < N; ++q) universe.emplace(ip->node_names[size_t(q)], q);
  PartIndex parts{*ip, {}};
  std::vector<ScenarioTables> tabs(NS);
  std::vector<std::vector<uint8_t>> member(NS);
  // the tables and members of stage x (chain stage g of its equivalent chain; prev: the stage before it, or NS)
  auto stage_tables = [&](size_t x, const ChainStage& cs, size_t g, size_t prev, const std::string& who) {
    tabs[x] = scenario_tables(*ip, model, flat[x], options, who, parts, g == 0);
    std::vector<uint8_t>& m = member[x];
    m.assign(size_t(N) + 1, 0);
    if (cs.NodesAll) {
      for (const auto& name : *cs.NodesAll) {
        auto it = universe.find(name);
        if (it == universe.end()) throw BlanceError(BLANCE_ERR_INVALID_ARG, "blance: " + who + "NodesAll name '" + name + "' is not in nodesAll");
        m[size_t(it->second)] = 1;
      }
    } else if (g == 0) {
      std::fill(m.begin(), m.begin() + N, uint8_t(1));
    } else {                           // (previous members - previous NodesToRemove) U NodesToAdd
      const std::vector<uint8_t>& pm = member[prev];
      const ScenarioTables& pt = tabs[prev];
      for (int32_t q = 0; q < N; ++q) m[size_t(q)] = (pm[size_t(q)] && !pt.removed[size_t(q)]) || tabs[x].added[size_t(q)];
    }
  };
  for (size_t i = 0; i < n; ++i)
    for (size_t t = 0; t < T; ++t)
      stage_tables(i * T + t, chains[i].Stages[t], t, i * T + t - 1, "chain " + std::to_string(i) + ", stage " + std::to_string(t) + ": ");
  for (size_t b = 0; b < nb; ++b) {
    const ChainBranch& br = (*branches)[b];
    for (size_t u = 0; u < TB; ++u) {
      const size_t x = n * T + b * TB + u, g = size_t(br.AfterStage + 1) + u;
      const size_t prev = u > 0 ? x - 1 : br.AfterStage >= 0 ? size_t(br.Chain) * T + size_t(br.AfterStage) : NS;
      stage_tables(x, br.Stages[u], g, prev, "branch " + std::to_string(b) + ", stage " + std::to_string(u) + ": ");
    }
  }
  std::vector<bool> want(NS, false);
  for (int i : wantMaps) {
    if (i < 0 || size_t(i) >= n) invalid("PlanNextMapChains: wantMaps index " + std::to_string(i) + " out of range");
    for (size_t t = 0; t < T; ++t) want[size_t(i) * T + t] = true;
  }
  for (size_t b = 0; b < nb; ++b)
    for (size_t u = 0; u < TB; ++u) want[n * T + b * TB + u] = (*branches)[b].WantMaps;
  std::vector<blance_chain_stage> stages(NS);
  std::vector<blance_scenario_opts> opts(stage_opts ? NS : n);
  std::vector<blance_scenario_out> out(NS);
  std::vector<blance_chain_out> net(n + nb);
  std::vector<std::vector<int64_t>> ops(NS, std::vector<int64_t>(size_t(NU) * 4 + 1)),
      load(NS, std::vector<int64_t>(size_t(S) * size_t(NU) + 1)), net_ops(n + nb, std::vector<int64_t>(size_t(NU) * 4 + 1));
  std::vector<std::unique_ptr<PlanOutBuffers>> maps(NS);
  for (size_t x = 0; x < NS; ++x) {
    const ScenarioTables& tb = tabs[x];
    stages[x] = blance_chain_stage{blance_scenario{tb.removed.data(), tb.added.data(), tb.add_is_nil, tb.has_node_weights,
                                                   tb.weight.data(), tb.has_weight.data()},
                                   member[x].data()};
    if (want[x]) maps[x] = std::make_unique<PlanOutBuffers>(*ip);
    out[x] = scenario_out(ops[x], load[x], maps[x].get());
  }
  // each stage's option groups, or the chain's when no stage sets its own (its stages then differ in node fields only)
  for (size_t x = 0; x < opts.size(); ++x) opts[x] = scenario_opts(tabs[stage_opts ? x : x * T]);
  for (size_t i = 0; i < n + nb; ++i) {
    net[i] = blance_chain_out{};
    net[i].node_ops = net_ops[i].data();
  }
  // the analyses (blance_plan_chains_exposure): per stage [n][T][nc], the net rebalance and the spans [n][nc]; the
  // branches' per stage [nb][TB][nc] and their nets [nb][nc] after them
  const size_t nc = scheduleConcurrency.size(), P = size_t(ip->in.n_parts);
  // every stage audits with its own rules
  AnalysisOutputs an(*ip, options, n * T, nc, audit, exposure, nc > 0, [&](size_t x) { return audit_rules(tabs[x], *ip); });
  AnalysisOutputs ban(*ip, options, nb * TB, nc, audit, exposure, false, [&](size_t x) { return audit_rules(tabs[n * T + x], *ip); });
  ScheduleBuffers net_sched((n + nb) * nc, size_t(NU));
  std::vector<std::unique_ptr<ExposureBuffers>> nebuf;
  std::vector<blance_exposure_out> neout;
  std::vector<std::unique_ptr<SpanBuffers>> sbuf;
  std::vector<blance_chain_span_out> sout;
  for (size_t x = 0; x < (n + nb) * nc; ++x) {
    if (exposure) {
      nebuf.push_back(std::make_unique<ExposureBuffers>(an.cap, an.eforest.names.size(), P));
      neout.push_back(nebuf.back()->out);
    }
    if (x >= n * nc) continue;
    sbuf.push_back(std::make_unique<SpanBuffers>(size_t(NU), P, an.eforest.names.size(), exposure != nullptr));
    sout.push_back(sbuf.back()->out);
  }
  std::vector<blance_chain_branch> br(nb);
  for (size_t b = 0; b < nb; ++b)
    br[b] = blance_chain_branch{(*branches)[b].Chain, (*branches)[b].AfterStage, stages.data() + n * T + b * TB, opts.data() + n * T + b * TB};
  blance_ctx* ctx = DefaultContext();
  // options per stage, or a schedule with options per chain: the two entry points take the same arguments
  auto* const analysed = stage_opts ? blance_plan_chains_ex : blance_plan_chains_exposure;
  const int st = nb ? blance_plan_chain_branches(
                          ctx, &ip->in, int32_t(n), int32_t(T), stages.data(), opts.data(), favorMinNodes ? 1 : 0, maxConcurrent,
                          int32_t(nc), nc ? scheduleConcurrency.data() : nullptr, nullptr, out.data(), net.data(),
                          nc ? an.sched.out.data() : nullptr, audit ? &an.forest.opts : nullptr, audit ? an.aout.data() : nullptr,
                          &an.eforest.opts, int32_t(an.cap), exposure ? an.eout.data() : nullptr, nc ? net_sched.out.data() : nullptr,
                          exposure ? neout.data() : nullptr, nc ? sout.data() : nullptr, int32_t(nb), int32_t(TB), br.data(),
                          out.data() + n * T, net.data() + n, nc ? ban.sched.out.data() : nullptr, audit ? ban.aout.data() : nullptr,
                          exposure ? ban.eout.data() : nullptr, nc ? net_sched.out.data() + n * nc : nullptr,
                          exposure ? neout.data() + n * nc : nullptr)
                 : stage_opts || nc
                     ? analysed(ctx, &ip->in, int32_t(n), int32_t(T), stages.data(), opts.data(), favorMinNodes ? 1 : 0, maxConcurrent,
                                int32_t(nc), nc ? scheduleConcurrency.data() : nullptr, nullptr, out.data(), net.data(),
                                nc ? an.sched.out.data() : nullptr, audit ? &an.forest.opts : nullptr, audit ? an.aout.data() : nullptr,
                                &an.eforest.opts, int32_t(an.cap), exposure ? an.eout.data() : nullptr, nc ? net_sched.out.data() : nullptr,
                                exposure ? neout.data() : nullptr, nc ? sout.data() : nullptr)
                     : blance_plan_chains(ctx, &ip->in, int32_t(n), int32_t(T), stages.data(), opts.data(), favorMinNodes ? 1 : 0,
                                          maxConcurrent, out.data(), net.data());
  if (st != BLANCE_OK) throw BlanceError(st, std::string("blance_plan_chains failed: ") + blance_last_error(ctx));
  // chain (or branch) i of n + nb: its stages' results from x0 on, its net and, for a chain, its span
  auto result = [&](size_t i, size_t x0, size_t len, AnalysisOutputs& a) {
    ChainResult c;
    for (size_t t = 0; t < len; ++t) {
      const size_t x = x0 + t;
      const int32_t* k = (tabs[x].set & BLANCE_OPT_CONSTRAINTS) ? tabs[x].constraints.data() : ip->state_constraints.data();
      ScenarioResult r = scenario_result(*ip, out[x], ops[x], load[x], maps[x].get(), k);
      a.name(*ip, i < n ? x : x - n * T, scheduleConcurrency, audit_rules(tabs[x], *ip).off, r);
      c.Stages.push_back(std::move(r));
    }
    c.NetNodeOps = node_ops_by_name(*ip, net_ops[i].data());
    c.NetOpsTotal = net[i].ops_total;
    c.NetPartsMoved = net[i].parts_moved;
    for (size_t k = 0; k < nc; ++k) {
      c.NetSchedules.push_back(name_schedule(*ip, net_sched.out[i * nc + k], scheduleConcurrency[k]));
      if (exposure) {
        nebuf[i * nc + k]->out = neout[i * nc + k];
        c.NetExposures.push_back(name_exposure(*nebuf[i * nc + k], an.cap, an.eforest.names, ip->part_names));
      }
      if (i >= n) continue;
      sbuf[i * nc + k]->out = sout[i * nc + k];
      c.Span.push_back(name_span(*ip, *sbuf[i * nc + k], scheduleConcurrency[k], an.eforest.names));
    }
    return c;
  };
  std::vector<ChainResult> res;
  for (size_t i = 0; i < n; ++i) res.push_back(result(i, i * T, T, an));
  if (branchResults) branchResults->clear();
  for (size_t b = 0; b < nb; ++b) branchResults->push_back(result(n + b, n * T + b * TB, TB, ban));
  return res;
}

// ------------------------------------------------------------------------------------
// CalcPartitionMoves

namespace {

struct MovesTables {
  Interner nodes;
  Strs state_names;      // visit states first, then the other keys that occur
  int32_t n_visit = 0;
  std::vector<int32_t> slot_off, beg_rows, end_rows;
  Strs part_names;
};

void intern_moves(const Strs& states, const std::vector<const NodesByState*>& begs,
                  const std::vector<const NodesByState*>& ends, MovesTables* t) {
  std::unordered_map<std::string, int32_t> sid;
  for (const auto& s : states) {
    if (sid.count(s)) invalid("CalcPartitionMoves: state '" + s + "' listed twice");
    sid[s] = int32_t(t->state_names.size());
    t->state_names.push_back(s);
  }
  t->n_visit = int32_t(states.size());
  static const NodesByState kEmptyNbs;
  auto scan = [&](const NodesByState* nbs, std::vector<int32_t>& cap) {
    if (!nbs) return;
    for (const auto& kv : *nbs) {
      auto it = sid.find(kv.first);
      if (it == sid.end()) { it = sid.emplace(kv.first, int32_t(t->state_names.size())).first; t->state_names.push_back(kv.first); cap.push_back(0); }
      cap[size_t(it->second)] = std::max(cap[size_t(it->second)], int32_t(deref(kv.second).size()));
    }
  };
  std::vector<int32_t> cap(t->state_names.size(), 0);
  for (auto* b : begs) scan(b, cap);
  for (auto* e : ends) scan(e, cap);
  const size_t S = t->state_names.size();
  t->slot_off.assign(S + 1, 0);
  for (size_t s = 0; s < S; ++s) t->slot_off[s + 1] = t->slot_off[s] + cap[s];
  const size_t SL = size_t(t->slot_off[S]), P = begs.size();
  t->beg_rows.assign(P * SL + 1, BLANCE_NO_NODE);
  t->end_rows.assign(P * SL + 1, BLANCE_NO_NODE);
  auto fill = [&](const NodesByState* nbs, int32_t* row) {
    if (!nbs) return;
    for (const auto& kv : *nbs) {
      int32_t slot = t->slot_off[size_t(sid.at(kv.first))];
      for (const auto& n : deref(kv.second)) row[slot++] = t->nodes.get(n);
    }
  };
  for (size_t p = 0; p < P; ++p) { fill(begs[p], t->beg_rows.data() + p * SL); fill(ends[p], t->end_rows.data() + p * SL); }
}

std::vector<std::vector<NodeStateOp>> run_moves(MovesTables& t, size_t P, bool favorMinNodes) {
  const size_t S = t.state_names.size(), SL = size_t(t.slot_off[S]);
  const int32_t max_ops = int32_t(std::max<size_t>(1, 2 * SL));
  std::vector<int32_t> op_node(P * size_t(max_ops) + 1), op_count(P + 1);
  std::vector<uint8_t> op_state(P * size_t(max_ops) + 1), op_kind(P * size_t(max_ops) + 1);
  blance_ctx* ctx = DefaultContext();
  int st = blance_calc_partition_moves(ctx, int32_t(P), int32_t(S), t.n_visit, t.slot_off.data(), t.beg_rows.data(),
                                       t.end_rows.data(), favorMinNodes ? 1 : 0, max_ops, op_node.data(),
                                       op_state.data(), op_kind.data(), op_count.data());
  if (st != BLANCE_OK) throw BlanceError(st, std::string("blance_calc_partition_moves failed: ") + blance_last_error(ctx));
  static const char* kOps[] = {"add", "del", "promote", "demote"};
  std::vector<std::vector<NodeStateOp>> out(P);
  for (size_t p = 0; p < P; ++p)
    for (int32_t i = 0; i < op_count[p]; ++i) {
      const size_t o = p * size_t(max_ops) + size_t(i);
      NodeStateOp op;
      op.Node = t.nodes.names[size_t(op_node[o])];
      op.State = op_state[o] == BLANCE_OP_STATE_NONE ? std::string() : t.state_names[op_state[o]];
      op.Op = kOps[op_kind[o]];
      out[p].push_back(std::move(op));
    }
  return out;
}

}  // namespace

std::vector<NodeStateOp> CalcPartitionMoves(const Strs& states, const NodesByState& beg, const NodesByState& end,
                                            bool favorMinNodes) {
  MovesTables t;
  intern_moves(states, {&beg}, {&end}, &t);
  return run_moves(t, 1, favorMinNodes)[0];
}

std::unordered_map<std::string, std::vector<NodeStateOp>> CalcPartitionMovesMap(
    const Strs& states, const PartitionMap& beg, const PartitionMap& end, bool favorMinNodes) {
  Strs names;
  std::unordered_set<std::string> seen;
  for (const auto& kv : beg) if (seen.insert(kv.first).second) names.push_back(kv.first);
  for (const auto& kv : end) if (seen.insert(kv.first).second) names.push_back(kv.first);
  std::sort(names.begin(), names.end());
  std::vector<const NodesByState*> begs, ends;
  for (const auto& n : names) {
    auto b = beg.find(n); auto e = end.find(n);
    begs.push_back(b == beg.end() ? nullptr : &b->second.NodesByState);
    ends.push_back(e == end.end() ? nullptr : &e->second.NodesByState);
  }
  MovesTables t;
  intern_moves(states, begs, ends, &t);
  auto ops = run_moves(t, names.size(), favorMinNodes);
  std::unordered_map<std::string, std::vector<NodeStateOp>> out;
  for (size_t p = 0; p < names.size(); ++p) out.emplace(names[p], std::move(ops[p]));
  return out;
}

namespace {

// The move lists of OrchestrateMoves(model, options, nodesAll, begMap, endMap) on the device and their lock-step
// schedule: what OrchestrateSchedule copies out and OrchestrateExposure counts over.
struct Orchestrated {
  MovesTables t;
  Strs names;                                        // partitions: begMap's keys in byte order
  blance_ctx* ctx = nullptr;
  std::unique_ptr<blance_moves, std::function<void(blance_moves*)>> h;
  int64_t total = 0;
  blance_schedule_out so{};
  void check(int st, const char* what) const {
    if (st != BLANCE_OK) throw BlanceError(st, std::string(what) + " failed: " + blance_last_error(ctx));
  }
};

std::unique_ptr<Orchestrated> orchestrate(const PartitionModel& model, const OrchestratorOptions& options, const Strs& nodesAll,
                                          const PartitionMap& begMap, const PartitionMap& endMap) {
  if (begMap.size() != endMap.size()) throw BlanceError(BLANCE_ERR_INVALID_ARG, "mismatched begMap and endMap");   // orchestrate.go:250-252
  auto o = std::make_unique<Orchestrated>();
  MovesTables& t = o->t;
  const Strs states = sort_state_names(model);
  for (const auto& kv : begMap) o->names.push_back(kv.first);   // orchestrate.go:273: the partitions of begMap
  std::sort(o->names.begin(), o->names.end());
  std::vector<const NodesByState*> begs, ends;
  for (const auto& n : o->names) {
    begs.push_back(&begMap.at(n).NodesByState);
    auto e = endMap.find(n);
    ends.push_back(e == endMap.end() ? nullptr : &e->second.NodesByState);
  }
  for (const auto& n : nodesAll) t.nodes.get(n);     // node ids: nodesAll first, so exactly they have a mover
  const size_t n_movers = t.nodes.names.size();
  intern_moves(states, begs, ends, &t);
  const int32_t P = int32_t(o->names.size()), S = int32_t(t.state_names.size()), NN = int32_t(t.nodes.names.size());
  std::vector<uint8_t> mover(size_t(NN) + 1, 0);
  for (size_t i = 0; i < n_movers; ++i) mover[i] = 1;
  o->ctx = DefaultContext();
  blance_ctx* ctx = o->ctx;
  blance_moves* h = nullptr;
  o->check(blance_moves_create(ctx, P, S, t.n_visit, t.slot_off.data(), t.beg_rows.data(), t.end_rows.data(),
                               options.FavorMinNodes ? 1 : 0, NN, &h, &o->total), "blance_moves_create");
  o->h = std::unique_ptr<blance_moves, std::function<void(blance_moves*)>>(h, [ctx](blance_moves* m) { blance_moves_free(ctx, m); });
  o->check(blance_moves_schedule(ctx, h, options.MaxConcurrentPartitionMovesPerNode, mover.data(), &o->so), "blance_moves_schedule");
  return o;
}

}  // namespace

std::vector<std::vector<AssignPartitionsCall>> OrchestrateSchedule(const PartitionModel& model, const OrchestratorOptions& options,
                                                                   const Strs& nodesAll, const PartitionMap& begMap,
                                                                   const PartitionMap& endMap) {
  const auto o = orchestrate(model, options, nodesAll, begMap, endMap);
  const MovesTables& t = o->t;
  const blance_schedule_out& so = o->so;
  const size_t P = o->names.size();
  std::vector<int64_t> round_off(size_t(so.rounds) + 1), sched(size_t(std::max<int64_t>(so.moves_done, 1)));
  o->check(blance_moves_schedule_fetch(o->ctx, o->h.get(), round_off.data(), sched.data()), "blance_moves_schedule_fetch");
  std::vector<int64_t> op_off(P + 1);
  std::vector<int32_t> op_node(size_t(std::max<int64_t>(o->total, 1)));
  std::vector<uint8_t> op_state(op_node.size()), op_kind(op_node.size());
  o->check(blance_moves_fetch(o->ctx, o->h.get(), op_off.data(), op_node.data(), op_state.data(), op_kind.data()), "blance_moves_fetch");
  static const char* kOps[] = {"add", "del", "promote", "demote"};
  std::vector<std::vector<AssignPartitionsCall>> out(size_t(so.rounds));
  for (size_t r = 0; r < out.size(); ++r)
    for (int64_t i = round_off[r]; i < round_off[r + 1]; ++i) {
      const int64_t op = sched[size_t(i)];
      const size_t p = size_t(std::upper_bound(op_off.begin(), op_off.end(), op) - op_off.begin()) - 1;
      const auto& node = t.nodes.names[size_t(op_node[size_t(op)])];
      if (out[r].empty() || out[r].back().Node != node) out[r].push_back(AssignPartitionsCall{node, {}, {}, {}});
      auto& call = out[r].back();
      call.Partitions.push_back(o->names[p]);
      call.States.push_back(op_state[size_t(op)] == BLANCE_OP_STATE_NONE ? std::string() : t.state_names[op_state[size_t(op)]]);
      call.Ops.push_back(kOps[op_kind[size_t(op)]]);
    }
  return out;
}

ExposureResult OrchestrateExposure(const PartitionModel& model, const OrchestratorOptions& options, const Strs& nodesAll,
                                   const PartitionMap& begMap, const PartitionMap& endMap,
                                   const std::optional<std::unordered_map<std::string, std::string>>& nodeHierarchy) {
  const auto o = orchestrate(model, options, nodesAll, begMap, endMap);
  const MovesTables& t = o->t;
  const size_t S = t.state_names.size(), P = o->names.size(), R1 = size_t(o->so.rounds) + 1;
  std::vector<int32_t> cons(S + 1, 0);               // the model's Constraints; 0 for states outside the model
  for (size_t s = 0; s < S; ++s) {
    auto it = model.find(t.state_names[s]);
    if (it != model.end()) cons[s] = it->second.Constraints;
  }
  const std::string top = top_priority_state_name(model);
  int32_t top_state = -1;
  for (size_t s = 0; s < S && !top.empty(); ++s)
    if (t.state_names[s] == top) top_state = int32_t(s);
  Forest f;
  build_forest(t.nodes.names, nodeHierarchy, false, &f);
  blance_exposure_in in{cons.data(), top_state, f.opts.n_domains, f.opts.domain_parent};
  ExposureBuffers b(R1, f.names.size(), P);
  o->check(blance_moves_exposure(o->ctx, o->h.get(), &in, &b.out), "blance_moves_exposure");
  return name_exposure(b, R1, f.names, o->names);
}

LoadResult OrchestrateLoad(const PartitionModel& model, const OrchestratorOptions& options, const Strs& nodesAll,
                           const PartitionMap& begMap, const PartitionMap& endMap,
                           const std::optional<std::unordered_map<std::string, int>>& partitionWeights) {
  const auto o = orchestrate(model, options, nodesAll, begMap, endMap);
  const MovesTables& t = o->t;
  const size_t S = t.state_names.size(), P = o->names.size(), NN = t.nodes.names.size(), K = (S + 1) * NN;
  std::vector<int32_t> weight(partitionWeights ? P : 0, 1);
  for (size_t p = 0; p < weight.size(); ++p) {
    auto it = partitionWeights->find(o->names[p]);
    if (it != partitionWeights->end()) weight[p] = it->second;
  }
  std::vector<int64_t> beg(std::max<size_t>(K, 1)), end(beg.size()), peak(beg.size());
  std::vector<int32_t> peak_round(beg.size());
  blance_load_in in{weight.empty() ? nullptr : weight.data(), nullptr};
  blance_load_out out{};
  out.node_beg = beg.data(); out.node_end = end.data(); out.node_peak = peak.data(); out.node_peak_round = peak_round.data();
  o->check(blance_moves_load(o->ctx, o->h.get(), &in, &out), "blance_moves_load");
  LoadResult r;
  r.Rounds = out.rounds;
  for (size_t s = 0; s <= S; ++s)
    for (size_t q = 0; q < NN; ++q) {
      const size_t i = s * NN + q;
      if (peak[i] == 0) continue;                    // the peak bounds both ends
      const NodeLoad l{beg[i], end[i], peak[i], peak_round[i]};
      if (s < S) r.States[t.state_names[s]][t.nodes.names[q]] = l;
      else r.Nodes[t.nodes.names[q]] = l;
    }
  r.OverMax = out.over_max;
  r.OverNode = out.over_node >= 0 ? t.nodes.names[size_t(out.over_node)] : std::string();
  r.KernelMs = out.kernel_ms;
  return r;
}

}  // namespace blance
