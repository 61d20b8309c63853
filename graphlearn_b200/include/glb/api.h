// Public C++ API of graphlearn_b200 (layer L7).
//
// The reference exposes Client / Server / Dataset / *Request / *Response classes from src/include/
// (client.h:33-80, server.h:30-60, dag_dataset.h:27-55, tensor.h:35-86); a C++ application links the shared object
// and drives sampling and lookups without Python.  This header is the equivalent surface for the GPU runtime: a C++
// program that links `graphlearn_b200/_C.so` (plus libtorch) gets
//
//   glb::api::Graph     in-HBM typed graph of ONE GPU: node tables + CSR topologies built from COO tensors or from the
//                       reference's table files (host_loader), with every operator the Client has - neighbour sampling
//                       (all strategies), full neighbours, degrees, attribute lookup, random walks, negative sampling,
//                       counts - each ONE kernel launch on the caller's CUDA stream (no request/response objects:
//                       tensors in, tensors out)
//   glb::api::Query     the GSL chain V(t).batch(B).shuffle().outV(e).sample(k).by(s)... as a value (the DagDef)
//   glb::api::Dataset   continuous execution of a Query into a ring of pre-allocated batches on a side stream
//                       (Tape/TapeStore, dag_dataset.h): Next() hands out batch i while batch i+1.. are being sampled;
//                       returns false at the end of an epoch (the reference's OutOfRange status)
//
// Multi-GPU jobs run one process per GPU through the Python runtime (symmetric heap + peer descriptors); this API is
// the single-GPU embedding surface (serving binaries, C++ trainers).  Everything is exported through pybind as
// `_C.CppGraph / _C.CppQuery / _C.CppDataset` as well so the test-suite can hold it against the Python path.
#pragma once
#include <ATen/ATen.h>
#include <c10/util/Optional.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

namespace glb {
namespace api {

enum class Strategy : int { kRandom = 0, kRandomWithoutReplacement = 1, kTopK = 2, kEdgeWeight = 3, kInDegree = 4 };

Strategy strategy_from_name(const std::string& name);

struct NodeTable {
  std::string type;
  int64_t num_nodes = 0;
  at::Tensor features;   // [n, d] fp32 / bf16 on the device (may be undefined)
  at::Tensor labels;     // [n] int64 (may be undefined)
  at::Tensor weights;    // [n] fp32 (may be undefined)
  at::Tensor desc;       // CPU int64 table descriptor consumed by the gather kernels
};

struct Topology {
  std::string type, src_type, dst_type;
  at::Tensor indptr, indices, eids, cumw, weights;   // rows sorted by weight descending (top-k == prefix)
  at::Tensor cumw_indeg;                              // built on demand for Strategy::kInDegree
  at::Tensor desc, desc_indeg;                        // CPU int64 CSR descriptors consumed by the sampling kernels
  int64_t num_edges = 0;
};

struct Stats {
  std::map<std::string, int64_t> node_count, edge_count;
};

class Graph {
 public:
  explicit Graph(int device_index = 0, int64_t seed = 0);

  // ---- construction (before Init); ids are dense [0, n) per node type
  Graph& AddNodes(const std::string& type, int64_t num_nodes, const c10::optional<at::Tensor>& features,
                  const c10::optional<at::Tensor>& labels = c10::nullopt, const c10::optional<at::Tensor>& weights = c10::nullopt,
                  bool store_bf16 = false);
  Graph& AddEdges(const std::string& type, const std::string& src_type, const std::string& dst_type, const at::Tensor& src,
                  const at::Tensor& dst, const c10::optional<at::Tensor>& weights = c10::nullopt);
  // reference table files ("id:int64 \t weight:float \t label:int64 \t feature:string"...), parsed by the native loader
  Graph& AddNodeFile(const std::string& type, const std::string& path, int64_t float_dim, bool weighted, bool labeled,
                     bool store_bf16 = false);
  Graph& AddEdgeFile(const std::string& type, const std::string& src_type, const std::string& dst_type, const std::string& path,
                     bool weighted);
  void Init();

  // ---- operators (Client::Sampling / GetDegree / LookupNodes / RandomWalk / ... )
  at::Tensor SampleNeighbors(const std::string& edge_type, const at::Tensor& ids, int64_t k, Strategy s = Strategy::kRandom,
                             const c10::optional<at::Tensor>& out = c10::nullopt, int64_t default_id = 0);
  // (values, offsets[B + 1]) of every neighbour
  std::vector<at::Tensor> FullNeighbors(const std::string& edge_type, const at::Tensor& ids);
  at::Tensor GetDegree(const std::string& edge_type, const at::Tensor& ids);
  at::Tensor LookupNodes(const std::string& node_type, const at::Tensor& ids, bool out_bf16 = false);
  at::Tensor LookupLabels(const std::string& node_type, const at::Tensor& ids);
  at::Tensor RandomWalk(const std::string& edge_type, const at::Tensor& ids, int64_t walk_len, double p = 1.0, double q = 1.0);
  at::Tensor NegativeSample(const std::string& edge_type, const at::Tensor& ids, int64_t k, bool strict = true,
                            bool by_in_degree = false);
  Stats GetStats() const;

  const NodeTable& nodes(const std::string& type) const;
  Topology& topology(const std::string& type);
  at::Device device() const { return device_; }
  at::Tensor rng_state() const { return rng_; }
  void AdvanceRng();
  bool initialized() const { return inited_; }

 private:
  void EnsureInDegree(Topology& t);
  at::Device device_;
  at::Tensor rng_;            // CUDA int64[2] {seed, offset}
  int64_t salt_ = 0;
  bool inited_ = false;
  std::map<std::string, NodeTable> nodes_;
  std::map<std::string, Topology> topo_;
  struct PendingEdges { std::string type, src_type, dst_type; at::Tensor src, dst, w; };
  std::vector<PendingEdges> pending_;
};

struct Hop {
  std::string edge_type;
  int64_t k;
  Strategy strategy;
  std::string alias;
};

class Query {
 public:
  static Query V(const std::string& node_type, const std::string& alias = "src");
  Query& Batch(int64_t batch_size);
  Query& Shuffle(bool traverse = true);
  Query& OutV(const std::string& edge_type, int64_t k, Strategy s = Strategy::kRandom, const std::string& alias = "");
  Query& WithFeatures(bool on = true);     // .values(): also look the feature rows of every hop up

  std::string node_type, root_alias;
  int64_t batch_size = 1;
  bool shuffle = false, features = false;
  std::vector<Hop> hops;
};

struct Batch {
  int64_t size = 0;                    // real seeds in this batch (the tail batch of an epoch may be short)
  std::vector<at::Tensor> ids;         // ids[0] = seeds [B], ids[i] = hop-i neighbours [B * k1 * .. * ki]
  std::vector<at::Tensor> features;    // same order (only with Query::WithFeatures)
  at::Tensor labels;                   // seed labels when the node table has labels
};

class Dataset {
 public:
  Dataset(std::shared_ptr<Graph> g, const Query& q, int64_t prefetch = 2, bool drop_last = false);
  ~Dataset();
  // false: the epoch is over (cursor rewinds, the next call starts the next epoch)
  bool Next(Batch* out);
  int64_t epoch() const { return epoch_; }
  int64_t batches_per_epoch() const;

 private:
  struct Impl;
  std::unique_ptr<Impl> impl_;
  int64_t epoch_ = 0;
};

}  // namespace api
}  // namespace glb
