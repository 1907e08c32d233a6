// memgraph_b200/csrc/mgp_module_common.hpp -- host-side pieces shared by the query modules (pagerank.so, gpu_bfs.so, ...):
// mgp_error -> exception with the reference's texts, owning iterator wrappers, the one-pass graph pull through
// the mgp_graph iterators (the reference's CreatePageRankGraph, mage/cpp/pagerank_module/pagerank_module.cpp:18-54),
// and the per-call glue around the algorithm: device choice, device-graph handles, rows and the error boundary.
#pragma once

#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "mgb200_bfs.h"
#include "mgb200_personalized.h"
#include "mgp_abi.h"

#ifdef MGB200_USE_REFERENCE_MGP_HEADER
// contract-check build against the reference header: keep the optional imports weak there too
extern "C" {
enum mgp_error mgp_result_reserve(struct mgp_result *res, size_t n) __attribute__((weak));
enum mgp_error mgp_log(enum mgp_log_level log_level, const char *output) __attribute__((weak));
int mgp_must_abort(struct mgp_graph *graph) __attribute__((weak));
}
#endif

namespace mgb200_module {

// ---- mgp_error -> exception, with the texts a user of the reference module would see ---------------
// (include/_mgp.hpp:25-56 maps codes to mg_exception types; include/mg_exceptions.hpp holds the texts.)
struct ModuleError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

inline const char *ErrorText(mgp_error code) {
  switch (code) {
    case mgp_error::MGP_ERROR_UNKNOWN_ERROR: return "Unknown exception!";
    case mgp_error::MGP_ERROR_UNABLE_TO_ALLOCATE:
      return "Could not allocate memory. For more details please visit https://memgr.ph/memory-control";
    case mgp_error::MGP_ERROR_INSUFFICIENT_BUFFER: return "Buffer is not sufficient to process procedure!";
    case mgp_error::MGP_ERROR_OUT_OF_RANGE: return "Index out of range!";
    case mgp_error::MGP_ERROR_LOGIC_ERROR: return "Logic exception, check the procedure signature!";
    case mgp_error::MGP_ERROR_DELETED_OBJECT: return "Object is deleted!";
    case mgp_error::MGP_ERROR_INVALID_ARGUMENT: return "Invalid argument!";
    case mgp_error::MGP_ERROR_KEY_ALREADY_EXISTS: return "Key you are trying to set already exists!";
    case mgp_error::MGP_ERROR_IMMUTABLE_OBJECT: return "Object you are trying to change is immutable!";
    case mgp_error::MGP_ERROR_VALUE_CONVERSION: return "Error in value conversion!";
    case mgp_error::MGP_ERROR_SERIALIZATION_ERROR: return "Error in serialization!";
    case mgp_error::MGP_ERROR_NOT_YET_IMPLEMENTED: return "Not yet implemented!";
    default: return nullptr;  // NO_ERROR and AUTHORIZATION_ERROR fall through in the reference as well
  }
}

inline void Check(mgp_error code) {
  if (const char *text = ErrorText(code)) throw ModuleError(text);
}

// Owning wrappers so no iterator / value leaks on any exit path (ownership rules: mg_procedure.h:887-920).
struct VerticesIt {
  mgp_vertices_iterator *it = nullptr;
  VerticesIt(mgp_graph *graph, mgp_memory *memory) { Check(mgp_graph_iter_vertices(graph, memory, &it)); }
  ~VerticesIt() {
    if (it) mgp_vertices_iterator_destroy(it);
  }
  mgp_vertex *Get() {
    mgp_vertex *v = nullptr;
    Check(mgp_vertices_iterator_get(it, &v));
    return v;
  }
  mgp_vertex *Next() {
    mgp_vertex *v = nullptr;
    Check(mgp_vertices_iterator_next(it, &v));
    return v;
  }
  VerticesIt(const VerticesIt &) = delete;
  VerticesIt &operator=(const VerticesIt &) = delete;
};

struct OutEdgesIt {
  mgp_edges_iterator *it = nullptr;
  OutEdgesIt(mgp_vertex *v, mgp_memory *memory) { Check(mgp_vertex_iter_out_edges(v, memory, &it)); }
  ~OutEdgesIt() {
    if (it) mgp_edges_iterator_destroy(it);
  }
  mgp_edge *Get() {
    mgp_edge *e = nullptr;
    Check(mgp_edges_iterator_get(it, &e));
    return e;
  }
  mgp_edge *Next() {
    mgp_edge *e = nullptr;
    Check(mgp_edges_iterator_next(it, &e));
    return e;
  }
  OutEdgesIt(const OutEdgesIt &) = delete;
  OutEdgesIt &operator=(const OutEdgesIt &) = delete;
};

struct OwnedValue {
  mgp_value *v = nullptr;
  ~OwnedValue() {
    if (v) mgp_value_destroy(v);
  }
};

// gid -> dense id, open addressing; a gid that was never visited resolves to dense id 0, which is
// what the reference's unordered_map::operator[] lookup yields (pagerank_module.cpp:50).
class GidMap {
 public:
  void Reserve(std::size_t n) {
    std::size_t cap = 16;
    while (cap < n * 2 + 2) cap <<= 1;
    keys_.assign(cap, 0);
    vals_.assign(cap, kEmpty);
    mask_ = cap - 1;
    size_ = 0;
  }
  void Put(int64_t gid, uint64_t dense) {
    if ((size_ + 1) * 2 > keys_.size()) Grow();
    Insert(gid, dense);
  }
  bool Find(int64_t gid, uint64_t *dense) const {
    if (keys_.empty()) return false;
    std::size_t i = Hash(gid) & mask_;
    while (vals_[i] != kEmpty) {
      if (keys_[i] == gid) {
        *dense = vals_[i];
        return true;
      }
      i = (i + 1) & mask_;
    }
    return false;
  }
  uint64_t GetOrZero(int64_t gid) const {
    if (keys_.empty()) return 0;
    std::size_t i = Hash(gid) & mask_;
    while (vals_[i] != kEmpty) {
      if (keys_[i] == gid) return vals_[i];
      i = (i + 1) & mask_;
    }
    return 0;
  }

 private:
  static constexpr uint64_t kEmpty = ~0ull;
  static std::size_t Hash(int64_t gid) {
    uint64_t z = static_cast<uint64_t>(gid) + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return static_cast<std::size_t>(z ^ (z >> 31));
  }
  void Insert(int64_t gid, uint64_t dense) {
    std::size_t i = Hash(gid) & mask_;
    while (vals_[i] != kEmpty) {
      if (keys_[i] == gid) {
        vals_[i] = dense;  // same gid visited again: last assignment wins, as with operator[]
        return;
      }
      i = (i + 1) & mask_;
    }
    keys_[i] = gid;
    vals_[i] = dense;
    ++size_;
  }
  void Grow() {
    std::vector<int64_t> old_keys;
    std::vector<uint64_t> old_vals;
    old_keys.swap(keys_);
    old_vals.swap(vals_);
    const std::size_t cap = old_keys.empty() ? 16 : old_keys.size() * 2;
    keys_.assign(cap, 0);
    vals_.assign(cap, kEmpty);
    mask_ = cap - 1;
    size_ = 0;
    for (std::size_t i = 0; i < old_keys.size(); ++i)
      if (old_vals[i] != kEmpty) Insert(old_keys[i], old_vals[i]);
  }
  std::vector<int64_t> keys_;
  std::vector<uint64_t> vals_;
  std::size_t mask_ = 0, size_ = 0;
};

struct HostGraph {
  std::vector<int64_t> gid_of_dense;  // reference id_to_memgraph (:42)
  std::vector<uint32_t> from, to;     // dense (source, destination) per edge, in iteration order; 32-bit: the device
                                      // labels are, and the pull is the place to narrow (half the host memory, no
                                      // second pass before the upload)
  GidMap dense_of_gid;                // reference memgraph_to_id
};

inline bool MustAbort(mgp_graph *graph) { return mgp_must_abort != nullptr && mgp_must_abort(graph) != 0; }

// What to do with an edge whose destination was never visited by the vertex iterator (possible in analytical mode):
//   kUnknownToZero  the reference PageRank quirk, kept for drop-in fidelity: operator[] maps it to dense id 0 (:50)
//   kUnknownDropped the edge is dropped -- for paths whose reference has no such quirk (BFS: a fabricated edge to the
//                   first vertex would change distances)
enum class UnknownGid { kUnknownToZero, kUnknownDropped };

// The reference's ingest (CreatePageRankGraph :18-54): one vertex iterator, one out-edge iterator per
// vertex, dense id = visit index, destinations remapped afterwards.
// Optional per-edge read in the same pass: `read(edge)` is called on every out-edge and its result lands in
// `*edge_values`, kept in step with hg.from / hg.to (dropped edges drop their value too).  Without it (the default)
// nothing is read and the function is the plain pull.
template <typename Value = int, typename Read = std::nullptr_t>
inline HostGraph PullGraph(mgp_graph *graph, mgp_memory *memory, UnknownGid policy = UnknownGid::kUnknownToZero,
                           Read read = nullptr, std::vector<Value> *edge_values = nullptr) {
  constexpr bool kRead = !std::is_same_v<Read, std::nullptr_t>;
  HostGraph hg;
  std::size_t approx_vertices = 0, approx_edges = 0;
  Check(mgp_graph_approximate_vertex_count(graph, &approx_vertices));
  Check(mgp_graph_approximate_edge_count(graph, &approx_edges));
  hg.gid_of_dense.reserve(approx_vertices);
  hg.from.reserve(approx_edges);
  std::vector<int64_t> to_gid;
  to_gid.reserve(approx_edges);
  GidMap &dense_of_gid = hg.dense_of_gid;
  dense_of_gid.Reserve(approx_vertices);

  VerticesIt vertices(graph, memory);
  for (mgp_vertex *source = vertices.Get(); source != nullptr; source = vertices.Next()) {
    mgp_vertex_id source_id{};
    Check(mgp_vertex_get_id(source, &source_id));
    const uint64_t source_dense = hg.gid_of_dense.size();
    if (source_dense >= 0xFFFFFFFEull) throw ModuleError("graph has more than 2^32 - 2 vertices");
    {
      OutEdgesIt edges(source, memory);
      for (mgp_edge *edge = edges.Get(); edge != nullptr; edge = edges.Next()) {
        mgp_vertex *destination = nullptr;
        Check(mgp_edge_get_to(edge, &destination));
        mgp_vertex_id destination_id{};
        Check(mgp_vertex_get_id(destination, &destination_id));
        hg.from.push_back(static_cast<uint32_t>(source_dense));
        to_gid.push_back(destination_id.as_int);
        if constexpr (kRead) edge_values->push_back(read(edge));
      }
    }
    dense_of_gid.Put(source_id.as_int, source_dense);
    hg.gid_of_dense.push_back(source_id.as_int);
    if ((source_dense & 0xFFF) == 0 && MustAbort(graph)) throw ModuleError("procedure aborted by the host");
  }
  // Reference quirk kept: `from` was recorded as the visit index, but the reference remaps the SOURCE
  // gid through the map as well (:50); the two differ only if a gid is visited twice, where the map
  // holds the later index.
  hg.to.resize(to_gid.size());
  std::size_t kept = 0;
  for (std::size_t e = 0; e < to_gid.size(); ++e) {
    uint64_t dst = 0;
    const bool known = dense_of_gid.Find(to_gid[e], &dst);
    if (!known && policy == UnknownGid::kUnknownDropped) continue;
    hg.from[kept] = static_cast<uint32_t>(dense_of_gid.GetOrZero(hg.gid_of_dense[hg.from[e]]));
    hg.to[kept] = static_cast<uint32_t>(known ? dst : 0);
    if constexpr (kRead) (*edge_values)[kept] = (*edge_values)[e];
    ++kept;
  }
  hg.from.resize(kept);
  hg.to.resize(kept);
  if constexpr (kRead) edge_values->resize(kept);
  return hg;
}

// ---- per-call glue: the device, the device-graph handles, the rows and the callback's error boundary ----------------

// The device a module's call runs on: MGB200_DEVICE, default 0.
inline int DeviceFromEnv() {
  const char *dev_env = std::getenv("MGB200_DEVICE");
  return dev_env ? std::atoi(dev_env) : 0;
}

// A device call's nonzero return code as a ModuleError with mgb200_last_error()'s text.  The text is copied into the
// exception before any handle is destroyed by the unwinding, so a destroy cannot overwrite it.
inline void CheckDevice(int rc) {
  if (rc != MGB200_OK) throw ModuleError(mgb200_last_error());
}

// The `should_abort` poll the device loops take: the host's mgp_must_abort for the graph passed as `user`.
inline int MustAbortPoll(void *user) { return MustAbort(static_cast<mgp_graph *>(user)) ? 1 : 0; }

// Owns one device-graph handle (null until a create call fills `h`); Release() hands it to an owner that outlives the
// call, such as the PageRank module's graph cache.
template <typename T, void (*Destroy)(T *)>
struct DeviceHandle {
  T *h = nullptr;
  DeviceHandle() = default;
  ~DeviceHandle() { Destroy(h); }
  T *Release() {
    T *released = h;
    h = nullptr;
    return released;
  }
  DeviceHandle(const DeviceHandle &) = delete;
  DeviceHandle &operator=(const DeviceHandle &) = delete;
};
using DeviceGraph = DeviceHandle<mgb200_graph, mgb200_graph_destroy>;
using BfsGraph = DeviceHandle<mgb200_bfs_graph, mgb200_bfs_graph_destroy>;
using HitsGraph = DeviceHandle<mgb200_hits_graph, mgb200_hits_graph_destroy>;

// A pulled graph uploaded as a BFS device graph on DeviceFromEnv().  The upload takes 64-bit endpoints, so the edges are
// widened once into `from` / `to`; biconnectivity and gpu_wsp pass the same arrays on to their later calls.
struct BfsDeviceGraph {
  std::vector<uint64_t> from, to;
  BfsGraph graph;
  explicit BfsDeviceGraph(const HostGraph &hg) : from(hg.from.begin(), hg.from.end()), to(hg.to.begin(), hg.to.end()) {
    CheckDevice(mgb200_bfs_graph_create_host(DeviceFromEnv(), hg.gid_of_dense.size(), from.size(), from.data(),
                                             to.data(), &graph.h));
  }
};

constexpr const char *kFieldNode = "node";

// The vertex `gid` as a value in *out; false when it has vanished in analytical mode (the row is skipped), "Invalid ID!"
// in transactional mode (mg_utility::GetNodeForInsertion).
inline bool NodeValue(mgp_graph *graph, mgp_memory *memory, int64_t gid, OwnedValue *out) {
  mgp_vertex *vertex = nullptr;
  Check(mgp_graph_get_vertex_by_id(graph, mgp_vertex_id{gid}, memory, &vertex));
  if (vertex == nullptr) {
    int transactional = 0;
    Check(mgp_graph_is_transactional(graph, &transactional));
    if (transactional) throw ModuleError("Invalid ID!");
    return false;
  }
  Check(mgp_value_make_vertex(vertex, &out->v));  // takes ownership of `vertex` on success
  return true;
}

inline mgp_result_record *NewRecord(mgp_result *result) {
  mgp_result_record *record = nullptr;
  Check(mgp_result_new_record(result, &record));
  if (record == nullptr)
    throw ModuleError("Not enough memory! For more details please visit https://memgr.ph/memory-control");
  return record;
}

inline void InsertColumns(mgp_result_record *, mgp_memory *) {}

// (name, value) pairs: a floating-point value becomes a FLOAT column, an integer an INTEGER column.  Only the mgp_value_make_*
// a module's columns need is instantiated, so a module imports nothing it does not use.
template <typename T, typename... Rest>
void InsertColumns(mgp_result_record *record, mgp_memory *memory, const char *field, T value, Rest... rest) {
  OwnedValue column;
  if constexpr (std::is_floating_point_v<T>) {
    Check(mgp_value_make_double(value, memory, &column.v));
  } else {
    static_assert(std::is_integral_v<T>);
    Check(mgp_value_make_int(value, memory, &column.v));
  }
  Check(mgp_result_record_insert(record, field, column.v));
  InsertColumns(record, memory, rest...);
}

// One row: `node` (the vertex `gid`), then the (name, value) columns in order.  No row when the vertex has vanished in
// analytical mode (NodeValue).
template <typename... Columns>
void EmitNodeRow(mgp_graph *graph, mgp_result *result, mgp_memory *memory, int64_t gid, Columns... columns) {
  OwnedValue node;
  if (!NodeValue(graph, memory, gid, &node)) return;
  mgp_result_record *record = NewRecord(result);
  Check(mgp_result_record_insert(record, kFieldNode, node.v));
  InsertColumns(record, memory, columns...);
}

// The procedure callback around `Body`: nothing may escape it, so an exception becomes the procedure's error message,
// which the engine reports as QueryRuntimeException("<module>.<procedure>: <message>").
template <void (*Body)(mgp_list *, mgp_graph *, mgp_result *, mgp_memory *)>
void Guarded(mgp_list *args, mgp_graph *graph, mgp_result *result, mgp_memory *memory) {
  try {
    Body(args, graph, result, memory);
  } catch (const std::exception &e) {
    (void)mgp_result_set_error_msg(result, e.what());
  } catch (...) {
    (void)mgp_result_set_error_msg(result, "Unknown exception!");
  }
}


}  // namespace mgb200_module
