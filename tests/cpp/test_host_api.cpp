// C++ host-API tests over libtncb200, written to read like the reference's own tests
// (tnc/src/tensornetwork/contraction.rs:226-264, io/qasm/qasm_importer.rs:171-194,
// builders/circuit_builder.rs:372-396, io/hdf5.rs:196-257).  Needs a GPU; run by tests/test_gpu_cpp_host.py.
// `test_host_api --io <dir>` runs only the HDF5 tests, which need no GPU (tests/test_gpu_cpp_host.py::test_cpp_hdf5_io).
// `test_host_api --deriv <dir>` writes the derivative methods' blocks (tests/test_gpu_general_networks.py).
#include <cmath>
#include <cstdio>
#include <cstring>
#include "tnc.hpp"

using namespace tnc;
static int failures = 0;
#define EXPECT(cond) do { if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #cond); failures++; } } while (0)
static bool approx(Complex64 a, Complex64 b, double eps = 4 * 2.220446049250313e-16) { return std::abs(a - b) <= eps; }

static void test_outer_product_contraction(Context& ctx) {
  Tensor t1({0}, {3}), t2({1}, {2});
  t1.set_tensor_data(TensorData::new_from_data({3}, {{1, 0}, {2, 5}, {3, -1}}));
  t2.set_tensor_data(TensorData::new_from_data({2}, {{-4, 2}, {0, -1}}));
  Tensor t3 = Tensor::new_composite({t1, t2});
  Tensor result = contract_tensor_network(ctx, std::move(t3), ContractionPath::single(0, 1));
  EXPECT((result.legs == std::vector<uint64_t>{1, 0}));
  EXPECT((result.bond_dims == std::vector<uint64_t>{2, 3}));
  const Complex64 ref[6] = {{-4, 2}, {-18, -16}, {-10, 10}, {0, -1}, {5, -2}, {-1, -3}};
  auto e = result.elements();
  for (int i = 0; i < 6; i++) EXPECT(e[i] == ref[i]);
}

static Tensor ket0(uint64_t edge) { Tensor t = Tensor::new_from_const({edge}, 2); t.set_tensor_data(TensorData::new_from_data({2}, {{1, 0}, {0, 0}})); return t; }
static Tensor gate(std::vector<uint64_t> legs, const char* name) { Tensor t = Tensor::new_from_const(std::move(legs), 2); t.set_tensor_data(TensorData::gate(name)); return t; }

static void test_bell_contract(Context& ctx) {
  // qreg q[2]; h q[0]; cx q[0], q[1];  statevector network, legs as Circuit::append_gate numbers them
  Tensor tn = Tensor::new_composite({ket0(0), ket0(1), gate({0, 2}, "h"), gate({2, 1, 3, 4}, "cx")});
  Tensor r = contract_tensor_network(ctx, std::move(tn), ContractionPath::simple({{0, 1}, {0, 2}, {0, 3}}));
  EXPECT((r.legs == std::vector<uint64_t>{3, 4}));
  auto e = r.elements();
  const double h = 0.70710678118654752440;
  EXPECT(approx(e[0], {h, 0}) && approx(e[1], {0, 0}) && approx(e[2], {0, 0}) && approx(e[3], {h, 0}));
}

static void test_hadamards_amplitude(Context& ctx) {
  std::vector<Tensor> ts;
  const int qubits = 5;
  for (int q = 0; q < qubits; q++) ts.push_back(ket0(q));
  for (int q = 0; q < qubits; q++) ts.push_back(gate({(uint64_t)q, (uint64_t)(qubits + q)}, "h"));
  for (int q = 0; q < qubits; q++) ts.push_back(ket0(qubits + q));  // <0| bras
  std::vector<std::pair<size_t, size_t>> p;
  for (size_t i = 1; i < ts.size(); i++) p.push_back({0, i});
  Tensor r = contract_tensor_network(ctx, Tensor::new_composite(ts), ContractionPath::simple(p));
  EXPECT(r.legs.empty());
  EXPECT(approx(r.elements()[0], {std::pow(0.70710678118654752440, qubits), 0}));
}

static void test_panics_become_errors(Context& ctx) {
  Tensor tn = Tensor::new_composite({ket0(0), gate({0, 1}, "h"), ket0(1)});
  try { contract_tensor_network(ctx, tn, ContractionPath::simple({{0, 1}, {2, 1}})); EXPECT(false); }
  catch (const Error& e) { EXPECT(e.status == TNCB_ERR_UNCONTRACTED); }
  try { contract_tensor_network(ctx, tn, ContractionPath::simple({{0, 1}})); EXPECT(false); }
  catch (const Error& e) { EXPECT(e.status == TNCB_ERR_NOT_CONTRACTED); }
  try { contract_tensor_network(ctx, Tensor::new_composite({ket0(0), gate({0, 1}, "foo"), ket0(1)}), ContractionPath::simple({{0, 1}, {0, 2}})); EXPECT(false); }
  catch (const Error& e) { EXPECT(e.status == TNCB_ERR_GATE && std::string(e.what()) == "Gate 'foo' not found."); }
}

static void test_nested(Context& ctx) {
  Tensor a = Tensor::new_composite({ket0(0), gate({0, 1}, "h")});
  Tensor b = Tensor::new_composite({ket0(1)});
  ContractionPath p; p.nested[0] = ContractionPath::single(0, 1); p.nested[1] = ContractionPath(); p.toplevel = {{0, 1}};
  Tensor r = contract_tensor_network(ctx, Tensor::new_composite({a, b}), p);
  EXPECT(approx(r.elements()[0], {0.70710678118654752440, 0}));
}

static void test_plan_and_repeated_calls(Context& ctx) {
  // the same 5-qubit Hadamard amplitude through a NetworkPlan (execute, stage + run) and through repeated direct calls
  // (second sighting compiles a cached plan): every route gives the identical value
  std::vector<Tensor> ts;
  const int qubits = 5;
  for (int q = 0; q < qubits; q++) ts.push_back(ket0(q));
  for (int q = 0; q < qubits; q++) ts.push_back(gate({(uint64_t)q, (uint64_t)(qubits + q)}, "h"));
  for (int q = 0; q < qubits; q++) ts.push_back(ket0(qubits + q));
  std::vector<std::pair<size_t, size_t>> p;
  for (size_t i = 1; i < ts.size(); i++) p.push_back({0, i});
  const Tensor tn = Tensor::new_composite(ts);
  const ContractionPath path = ContractionPath::simple(p);
  const Complex64 direct = contract_tensor_network(ctx, tn, path).elements()[0];
  NetworkPlan plan(ctx, tn, path);
  EXPECT(plan.execute(tn).elements()[0] == direct);
  plan.stage(tn);
  EXPECT(plan.run().elements()[0] == direct);
  EXPECT(plan.run().elements()[0] == direct);
  for (int rep = 0; rep < 3; rep++) EXPECT(contract_tensor_network(ctx, tn, path).elements()[0] == direct);
  ctx.set_tolerance(1e-10); ctx.set_tolerance(0.0);
}

// io/hdf5.rs:238-257 (test_write_read), :214-236 (test_load_tensor through a file this library wrote)
static void test_hdf5_write_read(const std::string& dir) {
  const std::vector<Complex64> data = {{1, 0}, {0, -2}, {-3, 0}, {-2, -1}, {0, 0}, {0.5, 2}};
  io::hdf5::store_data(dir + "/wr.h5", {2, 3}, data);
  std::vector<uint64_t> shape;
  auto read = io::hdf5::load_data(dir + "/wr.h5", &shape);
  EXPECT((shape == std::vector<uint64_t>{2, 3}));
  EXPECT(read == data);
  // a network file: "0" = [[1, 2i], [3, i]] with bids [0, 1]; "-1" without data, bids [0, 1]
  const std::vector<Complex64> m = {{1, 0}, {0, 2}, {3, 0}, {0, 1}};
  const char* names[2] = {"-1", "0"};
  const int ranks[2] = {0, 2};
  const uint64_t d0[2] = {2, 2}, bids[2] = {0, 1};
  const uint64_t* dims[2] = {nullptr, d0};
  const double* payload[2] = {nullptr, reinterpret_cast<const double*>(m.data())};
  const int64_t n_bids[2] = {2, 2};
  const uint64_t* all_bids[2] = {bids, bids};
  check(tncb_hdf5_store((dir + "/net.h5").c_str(), 2, names, ranks, dims, payload, n_bids, all_bids));
  Tensor tn = io::hdf5::load_tensor(dir + "/net.h5");
  EXPECT((tn.legs == std::vector<uint64_t>{0, 1}));
  EXPECT(tn.tensors.size() == 1);
  EXPECT((tn.tensor(0).legs == std::vector<uint64_t>{0, 1}) && (tn.tensor(0).bond_dims == std::vector<uint64_t>{2, 2}));
  EXPECT(tn.tensor(0).elements() == m);
  bool threw = false;
  try { io::hdf5::load_data(dir + "/missing.h5", &shape); } catch (const Error& e) { threw = e.status == TNCB_ERR_IO; }
  EXPECT(threw);
}

// builders::Circuit / Permutor: structure only (no GPU).  Leg numbering as circuit_builder.rs:184-277 produces it; the same
// circuit as test_bell_contract below builds by hand.
static void test_circuit_builder_structure() {
  using builders::Circuit; using builders::Permutor;
  Circuit c;
  auto q = c.allocate_register(2);
  c.append_gate(TensorData::gate("h"), {q[0]});
  c.append_gate(TensorData::gate("cx"), {q[0], q[1]});
  EXPECT(c.num_qubits() == 2);
  Circuit c2 = c;
  auto sv = std::move(c).into_statevector_network();
  const std::vector<std::vector<uint64_t>> legs = {{0}, {1}, {0, 2}, {2, 1, 3, 4}};
  EXPECT(sv.first.tensors.size() == 4);
  for (size_t i = 0; i < 4 && i < sv.first.tensors.size(); i++) {
    EXPECT(sv.first.tensor(i).legs == legs[i]);
    EXPECT(sv.first.tensor(i).bond_dims == std::vector<uint64_t>(legs[i].size(), 2));
  }
  EXPECT((sv.second.target_leg_order == std::vector<uint64_t>{3, 4}));
  EXPECT(sv.first.tensor(2).tensordata.kind == TensorData::Gate && sv.first.tensor(2).tensordata.gate_name == "h");
  auto amp = std::move(c2).into_amplitude_network("1*");
  EXPECT(amp.first.tensors.size() == 5 && (amp.first.tensor(4).legs == std::vector<uint64_t>{3}));
  EXPECT((amp.first.tensor(4).tensordata.matrix == std::vector<Complex64>{{0, 0}, {1, 0}}));
  EXPECT((amp.second.target_leg_order == std::vector<uint64_t>{4}));
  // expectation value network: 4 tensors, their adjoints on legs + 5, one Z per qubit
  Circuit c3; auto r = c3.allocate_register(2);
  c3.append_gate(TensorData::gate("h"), {r[0]}); c3.append_gate(TensorData::gate("cx"), {r[0], r[1]});
  Tensor ev = std::move(c3).into_expectation_value_network();
  EXPECT(ev.tensors.size() == 10);
  EXPECT((ev.tensor(7).legs == std::vector<uint64_t>{8, 9, 7, 6}) && ev.tensor(7).tensordata.adjoint);     // cx: halves swapped, + offset 5
  EXPECT((ev.tensor(8).legs == std::vector<uint64_t>{3, 8}) && ev.tensor(8).tensordata.gate_name == "z");
  EXPECT((ev.tensor(9).legs == std::vector<uint64_t>{4, 9}));
  // permutation_between (circuit_builder.rs:357-369)
  const std::vector<std::pair<std::vector<uint64_t>, std::vector<uint64_t>>> cases = {
      {{1, 2, 3, 4}, {1, 2, 3, 4}}, {{1, 2, 3, 4}, {4, 3, 2, 1}}, {{4, 3, 2, 1}, {1, 2, 3, 4}}, {{4, 1, 3, 2}, {2, 4, 3, 1}},
      {{5, 1, 4, 3, 2, 6}, {1, 6, 3, 5, 2, 4}}};
  for (auto& gt : cases) {
    auto p = Permutor::permutation_between(gt.first, gt.second);
    std::vector<uint64_t> applied;
    for (int i : p) applied.push_back(gt.first[i]);
    EXPECT(applied == gt.second);
  }
  bool threw = false;
  try { Circuit bad; auto b = bad.allocate_register(2); bad.append_gate(TensorData::gate("cx"), {b[0], b[0]}); } catch (const Error&) { threw = true; }
  EXPECT(threw);                                                  // "Qubit arguments must be unique"
}

// TensorData::File leaves (tensordata.rs:43-49) inside contract_tensor_network
static void test_file_leaf(Context& ctx, const std::string& dir) {
  const std::vector<Complex64> a = {{1, 0}, {2, 5}, {3, -1}}, b = {{-4, 2}, {0, -1}};
  io::hdf5::store_data(dir + "/a.h5", {3}, a);
  Tensor t1({0}, {3}), t2({1}, {2});
  t1.set_tensor_data(TensorData::file(dir + "/a.h5"));
  t2.set_tensor_data(TensorData::new_from_data({2}, b));
  Tensor result = contract_tensor_network(ctx, Tensor::new_composite({t1, t2}), ContractionPath::single(0, 1));
  const Complex64 ref[6] = {{-4, 2}, {-18, -16}, {-10, 10}, {0, -1}, {5, -2}, {-1, -3}};
  auto e = result.elements();
  for (int i = 0; i < 6; i++) EXPECT(e[i] == ref[i]);
}

// The derivative methods of NetworkPlan (ForGradients / vjp, ForTangents / jvp, ForHvp / hvp) on a nested network with
// mixed extents, a dim-1 leg, a single-leaf composite and a rank-2 result, with a wrt subset.  Payloads, tangents, seed
// and seed tangent come from small integer formulas (exact in double) that tests/test_gpu_general_networks.py
// reproduces; every block is written raw to <dir> and compared there bit for bit with the Python plans' results.
static Complex64 payload_at(size_t l, size_t e) { return {(double((7 * l + 3 * e) % 11) - 5.0) / 4.0, (double((5 * l + 2 * e) % 13) - 6.0) / 8.0}; }
static Complex64 tangent_at(size_t l, size_t e) { return {(double((3 * l + 5 * e) % 7) - 3.0) / 2.0, (double((l + 4 * e) % 9) - 4.0) / 4.0}; }
static Complex64 seed_at(size_t r) { return {(double((2 * r) % 5) - 2.0) / 2.0, (double((3 * r) % 7) - 3.0) / 4.0}; }
static Complex64 seed_tangent_at(size_t r) { return {(double((r + 1) % 3) - 1.0) / 2.0, (double((5 * r) % 4) - 1.5) / 2.0}; }

static Tensor formula_leaf(size_t l, std::vector<uint64_t> legs, std::vector<uint64_t> dims) {
  size_t n = 1;
  for (uint64_t d : dims) n *= d;
  std::vector<Complex64> x(n);
  for (size_t e = 0; e < n; e++) x[e] = payload_at(l, e);
  Tensor t(std::move(legs), dims);
  t.set_tensor_data(TensorData::new_from_data(dims, std::move(x)));
  return t;
}

static void write_block(const std::string& path, const std::vector<Complex64>& v) {
  FILE* f = std::fopen(path.c_str(), "wb");
  EXPECT(f != nullptr);
  if (!f) return;
  EXPECT(std::fwrite(v.data(), sizeof(Complex64), v.size(), f) == v.size());
  std::fclose(f);
}

static void test_derivative_methods(Context& ctx, const std::string& dir) {
  // leaves in depth-first order: L0 (0:3, 1:2, 9:2) L1 (1:2, 2:5, 3:1) | L2 (2:5, 4:3, 5:2) | L3 (4:3, 0:3, 6:2, 3:1) |
  // L4 (5:2, 7:7) L5 (7:7, 6:2, 8:3); open legs 9 and 8
  Tensor c0 = Tensor::new_composite({formula_leaf(0, {0, 1, 9}, {3, 2, 2}), formula_leaf(1, {1, 2, 3}, {2, 5, 1})});
  Tensor c1 = Tensor::new_composite({formula_leaf(2, {2, 4, 5}, {5, 3, 2})});
  Tensor l3 = formula_leaf(3, {4, 0, 6, 3}, {3, 3, 2, 1});
  Tensor c3 = Tensor::new_composite({formula_leaf(4, {5, 7}, {2, 7}), formula_leaf(5, {7, 6, 8}, {7, 2, 3})});
  const Tensor tn = Tensor::new_composite({c0, c1, l3, c3});
  ContractionPath path = ContractionPath::simple({{0, 1}, {0, 2}, {0, 3}});
  path.nested[0] = ContractionPath::single(0, 1);
  path.nested[1] = ContractionPath();
  path.nested[3] = ContractionPath::single(0, 1);
  const std::vector<size_t> wrt = {0, 2, 5};
  const size_t leaf_elems[6] = {12, 10, 30, 18, 14, 42};
  std::vector<Complex64> seed(6), seed_tangent(6);            // the result's 6 entries
  for (size_t r = 0; r < 6; r++) { seed[r] = seed_at(r); seed_tangent[r] = seed_tangent_at(r); }
  std::map<size_t, std::vector<Complex64>> tangents;
  for (size_t l : wrt) {
    tangents[l].resize(leaf_elems[l]);
    for (size_t e = 0; e < leaf_elems[l]; e++) tangents[l][e] = tangent_at(l, e);
  }
  {
    NetworkPlan plan(ctx, tn, path, NetworkPlan::ForGradients{wrt});
    plan.stage(tn);
    Tensor r = plan.run();
    EXPECT((r.bond_dims == std::vector<uint64_t>{3, 2}) || (r.bond_dims == std::vector<uint64_t>{2, 3}));
    write_block(dir + "/vjp_value.bin", r.elements());
    auto g = plan.vjp(seed);
    EXPECT(g.size() == wrt.size());
    for (auto& [l, v] : g) {
      EXPECT(v.size() == leaf_elems[l]);
      write_block(dir + "/vjp_" + std::to_string(l) + ".bin", v);
    }
  }
  {
    NetworkPlan plan(ctx, tn, path, NetworkPlan::ForTangents{wrt});
    plan.stage(tn);
    auto [value, tangent] = plan.jvp(tangents);
    write_block(dir + "/jvp_value.bin", value);
    write_block(dir + "/jvp_tangent.bin", tangent);
  }
  {
    NetworkPlan plan(ctx, tn, path, NetworkPlan::ForHvp{wrt});
    plan.stage(tn);
    auto h = plan.hvp(tangents, seed, seed_tangent);
    write_block(dir + "/hvp_value.bin", h.value);
    write_block(dir + "/hvp_tangent.bin", h.tangent);
    EXPECT(h.grads.size() == wrt.size() && h.grad_tangents.size() == wrt.size());
    for (auto& [l, v] : h.grads) write_block(dir + "/hvp_grad_" + std::to_string(l) + ".bin", v);
    for (auto& [l, v] : h.grad_tangents) write_block(dir + "/hvp_dgrad_" + std::to_string(l) + ".bin", v);
  }
}

int main(int argc, char** argv) {
  const std::string dir = argc > 2 ? argv[2] : "/tmp";
  if (argc > 1 && std::strcmp(argv[1], "--deriv") == 0) {           // ForGradients / ForTangents / ForHvp (GPU)
    try { Context ctx(0); test_derivative_methods(ctx, dir); } catch (const Error& e) { std::printf("FAIL uncaught tnc::Error %d: %s\n", e.status, e.what()); return 2; }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("HOST_DERIV_OK\n");
    return 0;
  }
  if (argc > 1 && std::strcmp(argv[1], "--io") == 0) {
    try { test_hdf5_write_read(dir); test_circuit_builder_structure(); } catch (const Error& e) { std::printf("FAIL uncaught tnc::Error %d: %s\n", e.status, e.what()); return 2; }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("HOST_IO_OK\n");
    return 0;
  }
  if (argc > 1 && std::strcmp(argv[1], "--file-leaf") == 0) {       // TensorData::File through the device path (GPU)
    try { Context ctx(0); test_file_leaf(ctx, dir); } catch (const Error& e) { std::printf("FAIL uncaught tnc::Error %d: %s\n", e.status, e.what()); return 2; }
    if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
    std::printf("HOST_FILE_LEAF_OK\n");
    return 0;
  }
  try {
    Context ctx(0);
    test_hdf5_write_read(dir);
    test_outer_product_contraction(ctx);
    test_bell_contract(ctx);
    test_hadamards_amplitude(ctx);
    test_panics_become_errors(ctx);
    test_nested(ctx);
    test_plan_and_repeated_calls(ctx);
  } catch (const Error& e) { std::printf("FAIL uncaught tnc::Error %d: %s\n", e.status, e.what()); return 2; }
  if (failures) { std::printf("%d failure(s)\n", failures); return 1; }
  std::printf("HOST_API_OK 7 tests\n");
  return 0;
}
