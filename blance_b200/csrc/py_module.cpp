// blance_b200/csrc/py_module.cpp — Python face of the host API (host_api.hpp), used
// by the tests and bench.py.  A PartitionMap crosses as
// {partitionName: {stateName: [node, ...] | None}} (Partition.Name == its key).
//
// PlanNextMapEx / CalcPartitionMoves here ARE the product path: they intern, call
// the CUDA library through the C ABI and un-intern.  InternedPlan / PlanOut expose
// the flat tables (and the address of the blance_plan_in / blance_plan_out structs)
// so that tests can hand the very same tables to the CPU oracle via ctypes.
#include <pybind11/numpy.h>
#include <chrono>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "host_api.hpp"

namespace py = pybind11;
using namespace blance;

using PyPartitionMap = std::unordered_map<std::string, NodesByState>;
using PyModel = std::unordered_map<std::string, std::pair<int, int>>;
using PyRules = std::unordered_map<std::string, std::vector<std::pair<int, int>>>;
using IntMap = std::unordered_map<std::string, int>;
using StrMap = std::unordered_map<std::string, std::string>;

static PartitionMap to_map(const PyPartitionMap& m) {
  PartitionMap out;
  out.reserve(m.size());
  for (const auto& kv : m) {
    Partition p;
    p.Name = kv.first;
    p.NodesByState = kv.second;
    out.emplace(kv.first, std::move(p));
  }
  return out;
}

static PyPartitionMap from_map(const PartitionMap& m) {
  PyPartitionMap out;
  out.reserve(m.size());
  for (const auto& kv : m) out[kv.first] = kv.second.NodesByState;
  return out;
}

static PartitionModel to_model(const PyModel& m) {
  PartitionModel out;
  for (const auto& kv : m) out[kv.first] = PartitionModelState{kv.second.first, kv.second.second};
  return out;
}

static PlanNextMapOptions to_options(const std::optional<IntMap>& msc, const std::optional<IntMap>& pw,
                                     const std::optional<IntMap>& ss, const std::optional<IntMap>& nw,
                                     const std::optional<StrMap>& nh, const std::optional<PyRules>& hr, int booster,
                                     int max_iterations, int engine) {
  PlanNextMapOptions o;
  o.ModelStateConstraints = msc;
  o.PartitionWeights = pw;
  o.StateStickiness = ss;
  o.NodeWeights = nw;
  o.NodeHierarchy = nh;
  if (hr) {
    HierarchyRules rules;
    for (const auto& kv : *hr) {
      auto& v = rules[kv.first];
      for (const auto& r : kv.second) v.push_back(HierarchyRule{r.first, r.second});
    }
    o.HierarchyRules = std::move(rules);
  }
  o.NodeScoreBooster = booster;
  o.MaxIterationsPerPlan = max_iterations;
  o.Engine = engine;
  return o;
}

template <class T>
static py::array_t<T> np_copy(const std::vector<T>& v, size_t n) {
  py::array_t<T> a(n);
  if (n) std::memcpy(a.mutable_data(), v.data(), sizeof(T) * n);
  return a;
}

static py::dict audit_dict(const MapAudit& a) {
  py::dict d;
  d["short_slots"] = a.ShortSlots; d["over_slots"] = a.OverSlots;
  d["rule_miss"] = a.RuleMiss; d["rule_tested"] = a.RuleTested;
  d["dom_top"] = a.DomTop; d["dom_all"] = a.DomAll; d["dom_copies"] = a.DomCopies;
  d["short_parts"] = a.ShortParts; d["rule_miss_parts"] = a.RuleMissParts; d["no_top_parts"] = a.NoTopParts;
  d["part_flags"] = a.PartFlags;
  if (a.HasFailoverSpread) {
    d["failover_spread"] = a.FailoverSpread;
    d["failover_max"] = py::make_tuple(a.FailoverMax, a.FailoverMaxFrom, a.FailoverMaxTo);
  }
  return d;
}

struct PyInterned { std::unique_ptr<InternedPlan> ip; };
struct PyOut { std::unique_ptr<PlanOutBuffers> ob; const InternedPlan* ip; };

PYBIND11_MODULE(_host, m) {
  m.doc() = "blance_b200 host API (C++ mirror of blance's api.go over the CUDA C ABI)";
  // a subclass of the pure-Python blance_b200.abi.BlanceError, so one except clause covers the ctypes face too
  py::register_exception<BlanceError>(m, "BlanceError", py::module_::import("blance_b200.abi").attr("BlanceError"));

  m.def(
      "PlanNextMapEx",
      [](const PyPartitionMap& prev, const std::optional<PyPartitionMap>& assign, const Strs& nodes_all,
         const OptStrs& nodes_to_remove, const OptStrs& nodes_to_add, const PyModel& model,
         const std::optional<IntMap>& msc, const std::optional<IntMap>& pw, const std::optional<IntMap>& ss,
         const std::optional<IntMap>& nw, const std::optional<StrMap>& nh, const std::optional<PyRules>& hr, int booster,
         int max_iterations, int engine) {
        PlanNextMapOptions o = to_options(msc, pw, ss, nw, nh, hr, booster, max_iterations, engine);
        PartitionMap prev_map = to_map(prev), assign_map;
        PartitionMap* assign_ptr = &prev_map;      // None = the same map object twice (plan_test.go:1716-1718)
        if (assign) { assign_map = to_map(*assign); assign_ptr = &assign_map; }
        Warnings warnings;
        PlanStats stats;
        PartitionMap next;
        {
          py::gil_scoped_release rel;
          next = PlanNextMapEx(prev_map, *assign_ptr, nodes_all, nodes_to_remove, nodes_to_add, to_model(model), o,
                               &warnings, &stats);
        }
        py::dict out;
        out["next_map"] = from_map(next);
        out["warnings"] = warnings;
        out["prev_map"] = from_map(prev_map);
        out["partitions_to_assign"] = from_map(*assign_ptr);
        out["iterations"] = stats.iters_run;
        out["converged"] = stats.converged;
        out["steps"] = stats.steps;
        out["device_ms"] = stats.device_ms;
        out["kernel_ms"] = stats.kernel_ms;
        out["pass_ms"] = stats.pass_ms;
        return out;
      },
      py::arg("prev_map"), py::arg("partitions_to_assign"), py::arg("nodes_all"), py::arg("nodes_to_remove"),
      py::arg("nodes_to_add"), py::arg("model"), py::arg("model_state_constraints") = py::none(),
      py::arg("partition_weights") = py::none(), py::arg("state_stickiness") = py::none(),
      py::arg("node_weights") = py::none(), py::arg("node_hierarchy") = py::none(),
      py::arg("hierarchy_rules") = py::none(), py::arg("booster") = 0, py::arg("max_iterations") = 10,
      py::arg("engine") = 0);

  // The string API end to end on a large synthetic cluster, without Python dicts in the way: the PartitionMap is
  // built here from flat rows with the naming recipe of blance_b200/synth.py (nodes "n%04d", partitions decimal,
  // states primary / replica / standby) - that is set-up, untimed - then PlanNextMapEx runs on it exactly as a Go
  // host would call it (maps of strings in, map of strings out, caller maps mutated).  Returns the stage times
  // and the next map turned back into rows so the caller can compare it with the flat path.
  m.def("bench_string_api", [](py::array_t<int32_t, py::array::c_style | py::array::forcecast> rows, int n_nodes,
                               std::vector<int> constraints, std::vector<int> removed, std::vector<int> added,
                               std::optional<py::array_t<int32_t, py::array::c_style | py::array::forcecast>> node_weights,
                               std::optional<py::array_t<int32_t, py::array::c_style | py::array::forcecast>> part_weight,
                               std::optional<py::array_t<uint8_t, py::array::c_style | py::array::forcecast>> part_has_weight,
                               std::optional<std::vector<int>> state_stickiness, int max_iterations) {
    static const char* kStates[] = {"primary", "replica", "standby"};
    const auto rb = rows.unchecked<2>();
    const ssize_t P = rb.shape(0), SL = rb.shape(1);
    const int S = (int)constraints.size();
    if (S > 3) throw std::runtime_error("bench_string_api: at most 3 states");
    Strs nodes((size_t)n_nodes);
    for (int i = 0; i < n_nodes; ++i) { char b[16]; std::snprintf(b, sizeof b, "n%04d", i); nodes[(size_t)i] = b; }
    PartitionModel model;
    for (int s = 0; s < S; ++s) model[kStates[s]] = PartitionModelState{s, constraints[(size_t)s]};
    PartitionMap prev;
    prev.reserve((size_t)P);
    for (ssize_t p = 0; p < P; ++p) {
      Partition part;
      part.Name = std::to_string(p);
      ssize_t slot = 0;
      for (int s = 0; s < S; ++s) {
        Strs l;
        for (int j = 0; j < constraints[(size_t)s]; ++j, ++slot)
          if (slot < SL && rb(p, slot) >= 0) l.push_back(nodes[(size_t)rb(p, slot)]);
        part.NodesByState[kStates[s]] = std::move(l);
      }
      prev.emplace(part.Name, std::move(part));
    }
    PlanNextMapOptions o;
    o.MaxIterationsPerPlan = max_iterations;
    if (node_weights) {
      o.NodeWeights.emplace();
      const auto w = node_weights->unchecked<1>();
      for (int i = 0; i < n_nodes; ++i) (*o.NodeWeights)[nodes[(size_t)i]] = w(i);
    }
    if (part_weight && part_has_weight) {
      o.PartitionWeights.emplace();
      const auto w = part_weight->unchecked<1>();
      const auto h = part_has_weight->unchecked<1>();
      for (ssize_t p = 0; p < P; ++p) if (h(p)) (*o.PartitionWeights)[std::to_string(p)] = w(p);
    }
    if (state_stickiness) {
      o.StateStickiness.emplace();
      for (int s = 0; s < S && s < (int)state_stickiness->size(); ++s) (*o.StateStickiness)[kStates[s]] = (*state_stickiness)[(size_t)s];
    }
    Strs rm, ad;
    for (int i : removed) rm.push_back(nodes[(size_t)i]);
    for (int i : added) ad.push_back(nodes[(size_t)i]);
    Warnings warnings;
    PlanStats stats;
    PartitionMap next;
    double total_ms;
    {
      py::gil_scoped_release rel;
      const auto t0 = std::chrono::steady_clock::now();
      next = PlanNextMapEx(prev, prev, nodes, OptStrs(rm), OptStrs(ad), model, o, &warnings, &stats);   // the same map twice, as blance's callers do
      total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    py::array_t<int32_t> out({P, SL});
    auto ob = out.mutable_unchecked<2>();
    for (ssize_t p = 0; p < P; ++p) for (ssize_t j = 0; j < SL; ++j) ob(p, j) = -1;
    for (const auto& kv : next) {
      const ssize_t p = std::stoll(kv.first);
      ssize_t slot = 0;
      for (int s = 0; s < S; ++s) {
        auto it = kv.second.NodesByState.find(kStates[s]);
        if (it != kv.second.NodesByState.end() && it->second)
          for (size_t j = 0; j < it->second->size() && (int)j < constraints[(size_t)s]; ++j) ob(p, slot + (ssize_t)j) = std::atoi((*it->second)[j].c_str() + 1);
        slot += constraints[(size_t)s];
      }
    }
    py::dict d;
    d["total_ms"] = total_ms; d["intern_ms"] = stats.intern_ms; d["call_ms"] = stats.call_ms;
    d["unintern_ms"] = stats.unintern_ms; d["mutate_ms"] = stats.mutate_ms; d["device_ms"] = stats.device_ms;
    d["iterations"] = stats.iters_run; d["steps"] = stats.steps; d["next_rows"] = out; d["warnings"] = (int)warnings.size();
    d["host_threads"] = HostThreads();
    return d;
  }, py::arg("rows"), py::arg("n_nodes"), py::arg("constraints"), py::arg("removed"), py::arg("added"),
     py::arg("node_weights") = py::none(), py::arg("part_weight") = py::none(), py::arg("part_has_weight") = py::none(),
     py::arg("state_stickiness") = py::none(), py::arg("max_iterations") = 10);

  m.def(
      "AuditMap",
      [](const PyPartitionMap& map, const Strs& nodes_all, const PyModel& model, const std::optional<IntMap>& msc,
         const std::optional<StrMap>& nh, const std::optional<PyRules>& hr, bool failover_spread) {
        PlanNextMapOptions o = to_options(msc, std::nullopt, std::nullopt, std::nullopt, nh, hr, 0, 10, 0);
        const PartitionMap pm = to_map(map);
        MapAudit a;
        {
          py::gil_scoped_release rel;
          a = AuditMap(pm, nodes_all, to_model(model), o, failover_spread);
        }
        return audit_dict(a);
      },
      py::arg("map"), py::arg("nodes_all"), py::arg("model"), py::arg("model_state_constraints") = py::none(),
      py::arg("node_hierarchy") = py::none(), py::arg("hierarchy_rules") = py::none(), py::arg("failover_spread") = false);

  m.def("CalcPartitionMoves", [](const Strs& states, const NodesByState& beg, const NodesByState& end, bool favor) {
    std::vector<std::tuple<std::string, std::string, std::string>> out;
    for (const auto& op : CalcPartitionMoves(states, beg, end, favor)) out.emplace_back(op.Node, op.State, op.Op);
    return out;
  });

  m.def("PartitionMapToJSON", [](const PyPartitionMap& m) { return py::bytes(PartitionMapToJSON(to_map(m))); },
        "the JSON wire form of a PartitionMap (api.go:30,35), byte for byte what Go's encoding/json emits");

  m.def("CalcPartitionMovesMap", [](const Strs& states, const PyPartitionMap& beg, const PyPartitionMap& end, bool favor) {
    std::unordered_map<std::string, std::vector<std::tuple<std::string, std::string, std::string>>> out;
    for (auto& kv : CalcPartitionMovesMap(states, to_map(beg), to_map(end), favor)) {
      auto& v = out[kv.first];
      for (const auto& op : kv.second) v.emplace_back(op.Node, op.State, op.Op);
    }
    return out;
  });

  m.def("OrchestrateSchedule", [](const PyModel& model, int max_concurrent, bool favor, const Strs& nodes_all,
                                  const PyPartitionMap& beg, const PyPartitionMap& end) {
    OrchestratorOptions o;
    o.MaxConcurrentPartitionMovesPerNode = max_concurrent;
    o.FavorMinNodes = favor;
    const PartitionMap b = to_map(beg), e = to_map(end);
    std::vector<std::vector<AssignPartitionsCall>> rounds;
    {
      py::gil_scoped_release rel;
      rounds = OrchestrateSchedule(to_model(model), o, nodes_all, b, e);
    }
    std::vector<std::vector<std::tuple<std::string, Strs, Strs, Strs>>> out(rounds.size());
    for (size_t r = 0; r < rounds.size(); ++r)
      for (auto& c : rounds[r]) out[r].emplace_back(c.Node, c.Partitions, c.States, c.Ops);
    return out;
  });

  m.def("OrchestrateExposure", [](const PyModel& model, int max_concurrent, bool favor, const Strs& nodes_all,
                                  const PyPartitionMap& beg, const PyPartitionMap& end, const std::optional<StrMap>& nh) {
    OrchestratorOptions o;
    o.MaxConcurrentPartitionMovesPerNode = max_concurrent;
    o.FavorMinNodes = favor;
    const PartitionMap b = to_map(beg), e = to_map(end);
    ExposureResult r;
    {
      py::gil_scoped_release rel;
      r = OrchestrateExposure(to_model(model), o, nodes_all, b, e, nh);
    }
    py::dict d;
    d["rounds"] = r.Rounds; d["series"] = r.Series; d["peak"] = r.Peak; d["peak_round"] = r.PeakRound; d["area"] = r.Area;
    d["dom_peak"] = r.DomPeak; d["dom_peak_round"] = r.DomPeakRound; d["part_min_copies"] = r.PartMinCopies;
    d["part_no_top"] = r.PartNoTop; d["part_flags"] = r.PartFlags; d["kernel_ms"] = r.KernelMs;
    return d;
  }, py::arg("model"), py::arg("max_concurrent"), py::arg("favor"), py::arg("nodes_all"), py::arg("beg"), py::arg("end"),
     py::arg("node_hierarchy") = py::none());

  py::class_<PyInterned>(m, "InternedPlan")
      .def_property_readonly("in_ptr", [](const PyInterned& s) { return (uintptr_t)&s.ip->in; })
      .def_property_readonly("n_nodes", [](const PyInterned& s) { return s.ip->in.n_nodes; })
      .def_property_readonly("n_node_ids", [](const PyInterned& s) { return s.ip->in.n_node_ids; })
      .def_property_readonly("n_states", [](const PyInterned& s) { return s.ip->in.n_states; })
      .def_property_readonly("n_parts", [](const PyInterned& s) { return s.ip->in.n_parts; })
      .def_property_readonly("n_slots", [](const PyInterned& s) { return s.ip->in.n_slots; })
      .def_property_readonly("n_rules", [](const PyInterned& s) { return s.ip->in.n_rules; })
      .def_property_readonly("n_hier_bits", [](const PyInterned& s) { return s.ip->in.n_hier_bits; })
      .def_property_readonly("node_names", [](const PyInterned& s) { return s.ip->node_names; })
      .def_property_readonly("state_names", [](const PyInterned& s) { return s.ip->state_names; })
      .def_property_readonly("part_names", [](const PyInterned& s) { return s.ip->part_names; })
      .def("set_engine", [](PyInterned& s, int e) { s.ip->in.engine = e; })
      .def("set_max_iters", [](PyInterned& s, int v) { s.ip->in.max_iters = v; })
      .def("tables", [](const PyInterned& s) {
        const InternedPlan& ip = *s.ip;
        py::dict d;
        d["state_priority"] = np_copy(ip.state_priority, ip.state_priority.size());
        d["state_constraints"] = np_copy(ip.state_constraints, ip.state_constraints.size());
        d["state_slot_off"] = np_copy(ip.state_slot_off, ip.state_slot_off.size());
        d["part_in_prev"] = np_copy(ip.part_in_prev, ip.part_in_prev.size());
        d["part_in_assign"] = np_copy(ip.part_in_assign, ip.part_in_assign.size());
        d["part_weight"] = np_copy(ip.part_weight, ip.part_weight.size());
        d["prev_rows"] = np_copy(ip.prev_rows, ip.prev_rows.size());
        d["cur_rows"] = np_copy(ip.cur_rows, ip.cur_rows.size());
        d["prev_shape"] = np_copy(ip.prev_shape, ip.prev_shape.size());
        d["cur_shape"] = np_copy(ip.cur_shape, ip.cur_shape.size());
        d["node_removed"] = np_copy(ip.node_removed, ip.node_removed.size());
        d["node_added"] = np_copy(ip.node_added, ip.node_added.size());
        d["ie_mask"] = np_copy(ip.ie_mask, ip.ie_mask.size());
        return d;
      });

  py::class_<PyOut>(m, "PlanOut")
      .def_property_readonly("out_ptr", [](const PyOut& s) { return (uintptr_t)&s.ob->out; })
      .def_property_readonly("next_rows", [](const PyOut& s) {
        return np_copy(s.ob->next_rows, (size_t)s.ip->in.n_parts * (size_t)s.ip->in.n_slots);
      })
      .def_property_readonly("next_shape", [](const PyOut& s) {
        return np_copy(s.ob->next_shape, (size_t)s.ip->in.n_parts * (size_t)s.ip->in.n_states);
      })
      .def_property_readonly("warn", [](const PyOut& s) {
        return np_copy(s.ob->warn, (size_t)s.ip->in.n_parts * (size_t)s.ip->in.n_states);
      })
      .def_property_readonly("iters_run", [](const PyOut& s) { return s.ob->out.iters_run; })
      .def_property_readonly("converged", [](const PyOut& s) { return s.ob->out.converged; })
      .def_property_readonly("steps", [](const PyOut& s) { return s.ob->out.steps; })
      .def_property_readonly("device_ms", [](const PyOut& s) { return s.ob->out.device_ms; })
      .def_property_readonly("kernel_ms", [](const PyOut& s) { return s.ob->out.kernel_ms; })
      .def_property_readonly("pass_ms", [](const PyOut& s) { return s.ob->out.pass_ms; });

  m.def(
      "intern_plan",
      [](const PyPartitionMap& prev, const std::optional<PyPartitionMap>& assign, const Strs& nodes_all,
         const OptStrs& nodes_to_remove, const OptStrs& nodes_to_add, const PyModel& model,
         const std::optional<IntMap>& msc, const std::optional<IntMap>& pw, const std::optional<IntMap>& ss,
         const std::optional<IntMap>& nw, const std::optional<StrMap>& nh, const std::optional<PyRules>& hr, int booster,
         int max_iterations, int engine) {
        PlanNextMapOptions o = to_options(msc, pw, ss, nw, nh, hr, booster, max_iterations, engine);
        PartitionMap prev_map = to_map(prev);
        PyInterned r;
        if (assign) r.ip = InternPlan(prev_map, to_map(*assign), nodes_all, nodes_to_remove, nodes_to_add, to_model(model), o);
        else r.ip = InternPlan(prev_map, prev_map, nodes_all, nodes_to_remove, nodes_to_add, to_model(model), o);
        return r;
      },
      py::arg("prev_map"), py::arg("partitions_to_assign"), py::arg("nodes_all"), py::arg("nodes_to_remove"),
      py::arg("nodes_to_add"), py::arg("model"), py::arg("model_state_constraints") = py::none(),
      py::arg("partition_weights") = py::none(), py::arg("state_stickiness") = py::none(),
      py::arg("node_weights") = py::none(), py::arg("node_hierarchy") = py::none(),
      py::arg("hierarchy_rules") = py::none(), py::arg("booster") = 0, py::arg("max_iterations") = 10,
      py::arg("engine") = 0);

  // what-if scenarios: (nodes_to_remove, nodes_to_add, then a (has_key, value) pair for each of node_weights,
  // model_state_constraints, state_stickiness, partition_weights, node_hierarchy, hierarchy_rules) per scenario;
  // has_key false inherits the options' value, a None value is nil
  using PyScenario = std::tuple<OptStrs, OptStrs, bool, std::optional<IntMap>, bool, std::optional<IntMap>, bool,
                                std::optional<IntMap>, bool, std::optional<IntMap>, bool, std::optional<StrMap>, bool,
                                std::optional<PyRules>>;
  auto to_scenarios = [](const std::vector<PyScenario>& v) {
    std::vector<Scenario> out;
    for (const auto& t : v) {
      Scenario s;
      s.NodesToRemove = std::get<0>(t);
      s.NodesToAdd = std::get<1>(t);
      if (std::get<2>(t)) s.NodeWeights = std::get<3>(t);
      if (std::get<4>(t)) s.ModelStateConstraints = std::get<5>(t);
      if (std::get<6>(t)) s.StateStickiness = std::get<7>(t);
      if (std::get<8>(t)) s.PartitionWeights = std::get<9>(t);
      if (std::get<10>(t)) s.NodeHierarchy = std::get<11>(t);
      if (std::get<12>(t)) {
        std::optional<HierarchyRules> rules;
        if (const auto& hr = std::get<13>(t)) {
          rules.emplace();
          for (const auto& kv : *hr) {
            auto& dst = (*rules)[kv.first];
            for (const auto& r : kv.second) dst.push_back(HierarchyRule{r.first, r.second});
          }
        }
        s.HierarchyRules = std::move(rules);
      }
      out.push_back(std::move(s));
    }
    return out;
  };

  m.def(
      "PlanNextMapScenarios",
      [to_scenarios](const PyPartitionMap& prev, const std::optional<PyPartitionMap>& assign, const Strs& nodes_all,
                     const PyModel& model, const std::vector<PyScenario>& scenarios, bool favor_min_nodes,
                     const std::vector<int>& want_maps, int max_concurrent, const std::optional<IntMap>& msc,
                     const std::optional<IntMap>& pw, const std::optional<IntMap>& ss, const std::optional<IntMap>& nw,
                     const std::optional<StrMap>& nh, const std::optional<PyRules>& hr, int booster, int max_iterations,
                     int engine, const std::vector<int>& schedule_concurrency, const std::optional<bool>& audit) {
        PlanNextMapOptions o = to_options(msc, pw, ss, nw, nh, hr, booster, max_iterations, engine);
        const PartitionMap prev_map = to_map(prev);
        const PartitionMap assign_map = assign ? to_map(*assign) : PartitionMap{};
        const std::vector<Scenario> scs = to_scenarios(scenarios);
        std::vector<ScenarioResult> res;
        ScenarioAudit aud;
        aud.FailoverSpread = audit.value_or(false);
        {
          py::gil_scoped_release rel;
          res = PlanNextMapScenarios(prev_map, assign ? assign_map : prev_map, nodes_all, to_model(model), o, scs,
                                     favor_min_nodes, want_maps, max_concurrent, schedule_concurrency, audit ? &aud : nullptr);
        }
        py::list out;
        for (const auto& r : res) {
          py::dict d;
          d["iterations"] = r.iters_run; d["converged"] = r.converged; d["steps"] = r.steps;
          d["sticky_steps"] = r.sticky_steps; d["parts_moved"] = r.parts_moved; d["ops_total"] = r.ops_total;
          d["warn_parts"] = r.warn_parts; d["node_ops"] = r.NodeOps; d["state_node_load"] = r.StateNodeLoad;
          if (r.HasMap) { d["next_map"] = from_map(r.NextMap); d["warnings"] = r.NextWarnings; }
          if (!schedule_concurrency.empty()) {
            py::list sl;
            for (const auto& s : r.Schedules) {
              py::dict sd;
              sd["MaxConcurrentPartitionMovesPerNode"] = s.MaxConcurrentPartitionMovesPerNode;
              sd["Rounds"] = s.Rounds; sd["MovesDone"] = s.MovesDone; sd["StuckParts"] = s.StuckParts;
              sd["MaxBatch"] = s.MaxBatch; sd["NodeRounds"] = s.NodeRounds; sd["NodeLastRound"] = s.NodeLastRound;
              sl.append(sd);
            }
            d["schedules"] = sl;
          }
          if (r.Audit) d["audit"] = audit_dict(*r.Audit);
          out.append(d);
        }
        return out;
      },
      py::arg("prev_map"), py::arg("partitions_to_assign"), py::arg("nodes_all"), py::arg("model"), py::arg("scenarios"),
      py::arg("favor_min_nodes") = false, py::arg("want_maps") = std::vector<int>{}, py::arg("max_concurrent") = 0,
      py::arg("model_state_constraints") = py::none(), py::arg("partition_weights") = py::none(),
      py::arg("state_stickiness") = py::none(), py::arg("node_weights") = py::none(), py::arg("node_hierarchy") = py::none(),
      py::arg("hierarchy_rules") = py::none(), py::arg("booster") = 0, py::arg("max_iterations") = 10, py::arg("engine") = 0,
      py::arg("schedule_concurrency") = std::vector<int>{}, py::arg("audit") = py::none());

  // chains: per chain (its option fields as a scenario tuple - the node sets are not read -, its stages); per stage
  // (nodes_to_remove, nodes_to_add, has_node_weights_key, node_weights, nodes_all or None for the default)
  using PyStage = std::tuple<OptStrs, OptStrs, bool, std::optional<IntMap>, OptStrs>;
  using PyChain = std::tuple<PyScenario, std::vector<PyStage>>;
  m.def(
      "PlanNextMapChains",
      [to_scenarios](const PyPartitionMap& prev, const std::optional<PyPartitionMap>& assign, const Strs& nodes_all,
                     const PyModel& model, const std::vector<PyChain>& chains, bool favor_min_nodes,
                     const std::vector<int>& want_maps, int max_concurrent, const std::optional<IntMap>& msc,
                     const std::optional<IntMap>& pw, const std::optional<IntMap>& ss, const std::optional<IntMap>& nw,
                     const std::optional<StrMap>& nh, const std::optional<PyRules>& hr, int booster, int max_iterations,
                     int engine) {
        PlanNextMapOptions o = to_options(msc, pw, ss, nw, nh, hr, booster, max_iterations, engine);
        const PartitionMap prev_map = to_map(prev);
        const PartitionMap assign_map = assign ? to_map(*assign) : PartitionMap{};
        std::vector<Chain> cs;
        for (const auto& c : chains) {
          Chain ch;
          ch.Options = to_scenarios({std::get<0>(c)})[0];
          for (const auto& st : std::get<1>(c)) {
            ChainStage s;
            s.NodesToRemove = std::get<0>(st);
            s.NodesToAdd = std::get<1>(st);
            if (std::get<2>(st)) s.NodeWeights = std::get<3>(st);
            s.NodesAll = std::get<4>(st);
            ch.Stages.push_back(std::move(s));
          }
          cs.push_back(std::move(ch));
        }
        std::vector<ChainResult> res;
        {
          py::gil_scoped_release rel;
          res = PlanNextMapChains(prev_map, assign ? assign_map : prev_map, nodes_all, to_model(model), o, cs, favor_min_nodes,
                                  want_maps, max_concurrent);
        }
        py::list out;
        for (const auto& c : res) {
          py::list stages;
          for (const auto& r : c.Stages) {
            py::dict d;
            d["iterations"] = r.iters_run; d["converged"] = r.converged; d["steps"] = r.steps;
            d["sticky_steps"] = r.sticky_steps; d["parts_moved"] = r.parts_moved; d["ops_total"] = r.ops_total;
            d["warn_parts"] = r.warn_parts; d["node_ops"] = r.NodeOps; d["state_node_load"] = r.StateNodeLoad;
            if (r.HasMap) { d["next_map"] = from_map(r.NextMap); d["warnings"] = r.NextWarnings; }
            stages.append(d);
          }
          py::dict net;
          net["node_ops"] = c.NetNodeOps; net["ops_total"] = c.NetOpsTotal; net["parts_moved"] = c.NetPartsMoved;
          py::dict d;
          d["stages"] = stages;
          d["net"] = net;
          out.append(d);
        }
        return out;
      },
      py::arg("prev_map"), py::arg("partitions_to_assign"), py::arg("nodes_all"), py::arg("model"), py::arg("chains"),
      py::arg("favor_min_nodes") = false, py::arg("want_maps") = std::vector<int>{}, py::arg("max_concurrent") = 0,
      py::arg("model_state_constraints") = py::none(), py::arg("partition_weights") = py::none(),
      py::arg("state_stickiness") = py::none(), py::arg("node_weights") = py::none(), py::arg("node_hierarchy") = py::none(),
      py::arg("hierarchy_rules") = py::none(), py::arg("booster") = 0, py::arg("max_iterations") = 10, py::arg("engine") = 0);

  // test hook: the blance_plan_in of scenario `index`, as an interned plan the CPU oracle can run
  m.def(
      "intern_scenario",
      [to_scenarios](const PyPartitionMap& prev, const std::optional<PyPartitionMap>& assign, const Strs& nodes_all,
                     const PyModel& model, const std::vector<PyScenario>& scenarios, size_t index,
                     const std::optional<IntMap>& msc, const std::optional<IntMap>& pw, const std::optional<IntMap>& ss,
                     const std::optional<IntMap>& nw, const std::optional<StrMap>& nh, const std::optional<PyRules>& hr,
                     int booster, int max_iterations, int engine) {
        PlanNextMapOptions o = to_options(msc, pw, ss, nw, nh, hr, booster, max_iterations, engine);
        const PartitionMap prev_map = to_map(prev);
        const PartitionMap assign_map = assign ? to_map(*assign) : PartitionMap{};
        PyInterned r;
        r.ip = InternScenario(prev_map, assign ? assign_map : prev_map, nodes_all, to_model(model), o, to_scenarios(scenarios), index);
        return r;
      },
      py::arg("prev_map"), py::arg("partitions_to_assign"), py::arg("nodes_all"), py::arg("model"), py::arg("scenarios"),
      py::arg("index"), py::arg("model_state_constraints") = py::none(), py::arg("partition_weights") = py::none(),
      py::arg("state_stickiness") = py::none(), py::arg("node_weights") = py::none(), py::arg("node_hierarchy") = py::none(),
      py::arg("hierarchy_rules") = py::none(), py::arg("booster") = 0, py::arg("max_iterations") = 10, py::arg("engine") = 0);

  // test hook: the fault-domain forest AuditMap builds over an interned plan's node ids
  m.def("audit_forest", [](const PyInterned& ip, const std::optional<StrMap>& nh) {
    Strs names;
    std::vector<int32_t> parent;
    AuditForest(*ip.ip, nh, &names, &parent);
    return py::make_tuple(names, parent);
  });

  m.def("plan_out", [](const PyInterned& ip) {
    PyOut o;
    o.ob = std::make_unique<PlanOutBuffers>(*ip.ip);
    o.ip = ip.ip.get();
    return o;
  }, py::keep_alive<0, 1>());

  // rows -> maps, with the caller-map mutation rule of plan.go:49-52 left to the caller
  m.def("unintern_plan", [](const PyInterned& ip, const PyOut& out) {
    Warnings w;
    PartitionMap next = UninternPlan(*ip.ip, *out.ob, &w);
    return py::make_tuple(from_map(next), w);
  });

  m.def("plan_result_to_json", [](const PyInterned& ip, const PyOut& out) { return py::bytes(PlanResultToJSON(*ip.ip, *out.ob)); },
        "rows of a plan result -> the JSON wire form of the next map, without building the PartitionMap");

  // the product C ABI on already-interned tables (GPU): returns the status code
  m.def("run_plan_cuda", [](const PyInterned& ip, PyOut& out) {
    blance_ctx* ctx = DefaultContext();
    int st;
    {
      py::gil_scoped_release rel;
      st = blance_plan_next_map(ctx, &ip.ip->in, &out.ob->out);
    }
    if (st != BLANCE_OK) throw BlanceError(st, std::string("blance_plan_next_map failed: ") + blance_last_error(ctx));
    return st;
  });

  m.def("ctx_ptr", []() { return (uintptr_t)DefaultContext(); });
  m.def("set_host_threads", [](int n) { SetHostThreads(n); });
  m.def("host_threads", []() { return HostThreads(); });
}
