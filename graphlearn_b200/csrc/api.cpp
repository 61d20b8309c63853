// Implementation of the public C++ API (include/glb/api.h): a single-GPU graph + GSL-style query + prefetching dataset
// on top of the same kernel launchers the Python runtime uses (sampling.cu, walk.cu, negative.cu, gather.cu,
// host_loader.cpp).  Reference surface: graphlearn/src/include/{client,server,dag_dataset}.h.
#include "glb/api.h"

#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAEvent.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/extension.h>

#include <stdexcept>

namespace glb {
// kernel launchers defined in the .cu files of this extension
std::vector<at::Tensor> sample_neighbors(const at::Tensor&, const at::Tensor&, int64_t, int64_t, int64_t, const c10::optional<at::Tensor>&, bool,
                                         int64_t, int64_t, const at::Tensor&, int64_t, bool, const c10::optional<at::Tensor>&);
at::Tensor get_degrees(const at::Tensor&, const at::Tensor&, int64_t);
std::vector<at::Tensor> sample_full(const at::Tensor&, const at::Tensor&, int64_t, bool, int64_t);
void rng_advance(const at::Tensor&, int64_t);
at::Tensor random_walk(const at::Tensor&, const at::Tensor&, int64_t, double, double, int64_t, int64_t, const at::Tensor&, int64_t);
at::Tensor negative_sample(const at::Tensor&, const at::Tensor&, int64_t, const c10::optional<at::Tensor>&, const at::Tensor&, int64_t, bool,
                           int64_t, int64_t, const at::Tensor&, int64_t, const c10::optional<at::Tensor>&);
at::Tensor gather_rows(const at::Tensor&, const at::Tensor&, bool, double);
std::vector<at::Tensor> load_table(const std::string&, bool, bool, bool, bool, std::vector<int64_t>, std::vector<int64_t>, const std::string&,
                                   const std::string&, int64_t, int64_t, int64_t);

namespace api {

namespace {
constexpr int kMaxWorld = 8;

at::Tensor csr_desc(const Topology& t, int64_t n_rows, const at::Tensor& cumw) {
  // layout of csrc/sampling.cu::csr_from_desc: [world, nrows[8], indptr[8], indices[8], eids[8], cumw[8], ts[8]]
  auto d = at::zeros({1 + 6 * kMaxWorld}, at::kLong);
  int64_t* p = d.data_ptr<int64_t>();
  p[0] = 1;
  p[1] = n_rows;
  p[1 + kMaxWorld] = reinterpret_cast<int64_t>(t.indptr.data_ptr());
  p[1 + 2 * kMaxWorld] = reinterpret_cast<int64_t>(t.indices.data_ptr());
  p[1 + 3 * kMaxWorld] = t.eids.defined() ? reinterpret_cast<int64_t>(t.eids.data_ptr()) : 0;
  p[1 + 4 * kMaxWorld] = cumw.defined() ? reinterpret_cast<int64_t>(cumw.data_ptr()) : 0;
  return d;
}

at::Tensor table_desc(const at::Tensor& feat) {
  // layout of csrc/host_utils.h::table_from_desc: [world, dim, stride, dtype code, nrows[8], base[8]]
  auto d = at::zeros({4 + 2 * kMaxWorld}, at::kLong);
  int64_t* p = d.data_ptr<int64_t>();
  p[0] = 1; p[1] = feat.size(1); p[2] = feat.stride(0); p[3] = feat.scalar_type() == at::kFloat ? 0 : 1;
  p[4] = feat.size(0);
  p[4 + kMaxWorld] = reinterpret_cast<int64_t>(feat.data_ptr());
  return d;
}

// per-row inclusive prefix sums of `w` (rows given by indptr) - the inverse-CDF table of the weighted samplers
at::Tensor row_cumsum(const at::Tensor& w, const at::Tensor& indptr) {
  if (w.numel() == 0) return w.clone();
  auto c = w.cumsum(0);
  auto starts = indptr.slice(0, 0, indptr.size(0) - 1);
  auto deg = indptr.slice(0, 1) - starts;
  auto before = at::cat({at::zeros({1}, c.options()), c}).index_select(0, starts);   // cumulative weight before each row
  return c - at::repeat_interleave(before, deg);
}
}  // namespace

Strategy strategy_from_name(const std::string& n) {
  if (n == "random") return Strategy::kRandom;
  if (n == "random_without_replacement") return Strategy::kRandomWithoutReplacement;
  if (n == "topk") return Strategy::kTopK;
  if (n == "edge_weight") return Strategy::kEdgeWeight;
  if (n == "in_degree") return Strategy::kInDegree;
  throw std::invalid_argument("unknown sampling strategy: " + n);
}

Graph::Graph(int device_index, int64_t seed) : device_(at::kCUDA, (c10::DeviceIndex)device_index) {
  rng_ = at::zeros({2}, at::TensorOptions().dtype(at::kLong).device(device_));
  rng_.select(0, 0).fill_(seed);
}

Graph& Graph::AddNodes(const std::string& type, int64_t num_nodes, const c10::optional<at::Tensor>& features,
                       const c10::optional<at::Tensor>& labels, const c10::optional<at::Tensor>& weights, bool store_bf16) {
  TORCH_CHECK(!inited_, "AddNodes after Init");
  NodeTable t;
  t.type = type;
  t.num_nodes = num_nodes;
  if (features.has_value() && features->defined()) {
    TORCH_CHECK(features->dim() == 2 && features->size(0) == num_nodes, "features must be [num_nodes, d]");
    auto f = features->to(device_, store_bf16 ? at::kBFloat16 : at::kFloat);
    // rows padded to a 16-byte multiple so that the 128-bit row loads of the gather kernels stay aligned
    const int64_t per16 = store_bf16 ? 8 : 4;
    const int64_t stride = (f.size(1) + per16 - 1) / per16 * per16;
    auto buf = at::zeros({num_nodes, stride}, f.options());
    buf.slice(1, 0, f.size(1)).copy_(f);
    t.features = buf.slice(1, 0, f.size(1));
    t.desc = table_desc(t.features);
  }
  if (labels.has_value() && labels->defined()) t.labels = labels->to(device_, at::kLong).contiguous();
  if (weights.has_value() && weights->defined()) t.weights = weights->to(device_, at::kFloat).contiguous();
  nodes_[type] = t;
  return *this;
}

Graph& Graph::AddEdges(const std::string& type, const std::string& src_type, const std::string& dst_type, const at::Tensor& src,
                       const at::Tensor& dst, const c10::optional<at::Tensor>& weights) {
  TORCH_CHECK(!inited_, "AddEdges after Init");
  TORCH_CHECK(src.numel() == dst.numel(), "src / dst length mismatch");
  PendingEdges e{type, src_type, dst_type, src.to(device_, at::kLong).contiguous(), dst.to(device_, at::kLong).contiguous(), at::Tensor()};
  if (weights.has_value() && weights->defined()) e.w = weights->to(device_, at::kFloat).contiguous();
  pending_.push_back(e);
  return *this;
}

Graph& Graph::AddNodeFile(const std::string& type, const std::string& path, int64_t float_dim, bool weighted, bool labeled, bool store_bf16) {
  // load_table returns [a, b, weights, labels, timestamps, int_attrs, float_attrs, str_blob, str_offsets]; attribute
  // type code 1 = float.  Ids must be dense 0..n-1 for this API.
  auto cols = glb::load_table(path, false, weighted, labeled, false, std::vector<int64_t>((size_t)float_dim, 1), {}, ":", "\t", 4, 0, 1);
  auto ids = cols[0];
  const int64_t n = ids.numel();
  auto order = ids.argsort();
  TORCH_CHECK(n == 0 || (ids.index_select(0, order).equal(at::arange(n, ids.options()))), "node ids of ", path, " are not dense 0..n-1");
  auto pick = [&](const at::Tensor& c) { return c.defined() && c.numel() ? c.index_select(0, order) : at::Tensor(); };
  c10::optional<at::Tensor> f, l, w;
  if (float_dim > 0) f = pick(cols[6]);
  if (labeled) l = pick(cols[3]);
  if (weighted) w = pick(cols[2]);
  return AddNodes(type, n, f, l, w, store_bf16);
}

Graph& Graph::AddEdgeFile(const std::string& type, const std::string& src_type, const std::string& dst_type, const std::string& path,
                          bool weighted) {
  auto cols = glb::load_table(path, true, weighted, false, false, {}, {}, ":", "\t", 4, 0, 1);
  c10::optional<at::Tensor> w;
  if (weighted) w = cols[2];
  return AddEdges(type, src_type, dst_type, cols[0], cols[1], w);
}

void Graph::Init() {
  TORCH_CHECK(!inited_, "Init called twice");
  c10::cuda::CUDAGuard guard(device_);
  for (auto& e : pending_) {
    TORCH_CHECK(nodes_.count(e.src_type) && nodes_.count(e.dst_type), "edge type ", e.type, " references an unknown node type");
    const int64_t n_src = nodes_[e.src_type].num_nodes;
    Topology t;
    t.type = e.type; t.src_type = e.src_type; t.dst_type = e.dst_type;
    t.num_edges = e.src.numel();
    // rows grouped by source; inside a row by weight descending (top-k is then a prefix, SURVEY O3)
    at::Tensor order;
    if (e.w.defined()) {
      auto by_w = e.w.argsort(/*stable=*/true, 0, /*descending=*/true);
      order = by_w.index_select(0, e.src.index_select(0, by_w).argsort(/*stable=*/true, 0, false));
    } else {
      order = e.src.argsort(/*stable=*/true, 0, false);
    }
    t.indices = e.dst.index_select(0, order).contiguous();
    t.eids = order.contiguous();
    auto counts = at::bincount(e.src, {}, n_src);
    t.indptr = at::cat({at::zeros({1}, counts.options()), counts.cumsum(0)}).contiguous();
    if (e.w.defined()) {
      t.weights = e.w.index_select(0, order).contiguous();
      t.cumw = row_cumsum(t.weights, t.indptr).contiguous();
    }
    t.desc = csr_desc(t, n_src, t.cumw);
    topo_[e.type] = t;
  }
  pending_.clear();
  inited_ = true;
}

void Graph::EnsureInDegree(Topology& t) {
  if (t.desc_indeg.defined()) return;
  auto indeg = at::bincount(t.indices, {}, nodes_.at(t.dst_type).num_nodes).to(at::kFloat);
  t.cumw_indeg = row_cumsum(indeg.index_select(0, t.indices), t.indptr).contiguous();
  t.desc_indeg = csr_desc(t, nodes_.at(t.src_type).num_nodes, t.cumw_indeg);
}

const NodeTable& Graph::nodes(const std::string& type) const {
  auto it = nodes_.find(type);
  TORCH_CHECK(it != nodes_.end(), "unknown node type ", type);
  return it->second;
}

Topology& Graph::topology(const std::string& type) {
  auto it = topo_.find(type);
  TORCH_CHECK(it != topo_.end(), "unknown edge type ", type);
  return it->second;
}

void Graph::AdvanceRng() { glb::rng_advance(rng_, 1); }

at::Tensor Graph::SampleNeighbors(const std::string& edge_type, const at::Tensor& ids, int64_t k, Strategy s,
                                  const c10::optional<at::Tensor>& out, int64_t default_id) {
  TORCH_CHECK(inited_, "Graph::Init has not been called");
  auto& t = topology(edge_type);
  const at::Tensor* desc = &t.desc;
  int64_t code = (int64_t)s;
  if (s == Strategy::kInDegree) { EnsureInDegree(t); desc = &t.desc_indeg; code = (int64_t)Strategy::kEdgeWeight; }
  if (s == Strategy::kEdgeWeight) TORCH_CHECK(t.cumw.defined(), "edge type ", edge_type, " has no weights");
  auto r = glb::sample_neighbors(*desc, ids.to(device_, at::kLong), k, code, /*filter_mode=*/0, c10::nullopt, /*padding_circular=*/true,
                                 /*retry=*/2, default_id, rng_, ++salt_, /*want_eids=*/false, out);
  return r[0];
}

std::vector<at::Tensor> Graph::FullNeighbors(const std::string& edge_type, const at::Tensor& ids) {
  auto& t = topology(edge_type);
  auto r = glb::sample_full(t.desc, ids.to(device_, at::kLong), /*cap=*/-1, /*want_eids=*/false, /*max_total=*/0);
  return {r[0], r[2]};
}

at::Tensor Graph::GetDegree(const std::string& edge_type, const at::Tensor& ids) {
  return glb::get_degrees(topology(edge_type).desc, ids.to(device_, at::kLong), /*cap=*/-1);
}

at::Tensor Graph::LookupNodes(const std::string& node_type, const at::Tensor& ids, bool out_bf16) {
  const auto& t = nodes(node_type);
  TORCH_CHECK(t.features.defined(), "node type ", node_type, " has no float attributes");
  return glb::gather_rows(t.desc, ids.to(device_, at::kLong), out_bf16, 0.0);
}

at::Tensor Graph::LookupLabels(const std::string& node_type, const at::Tensor& ids) {
  const auto& t = nodes(node_type);
  TORCH_CHECK(t.labels.defined(), "node type ", node_type, " has no labels");
  auto v = ids.to(device_, at::kLong);
  auto ok = (v >= 0).logical_and(v < t.num_nodes);
  return at::where(ok, t.labels.index_select(0, v.clamp(0, std::max<int64_t>(t.num_nodes - 1, 0)).view({-1})).view(v.sizes()),
                   at::full_like(v, -1));
}

at::Tensor Graph::RandomWalk(const std::string& edge_type, const at::Tensor& ids, int64_t walk_len, double p, double q) {
  auto& t = topology(edge_type);
  return glb::random_walk(t.desc, ids.to(device_, at::kLong), walk_len, p, q, /*default_id=*/-1, /*full_nbr_num=*/100, rng_, ++salt_);
}

at::Tensor Graph::NegativeSample(const std::string& edge_type, const at::Tensor& ids, int64_t k, bool strict, bool by_in_degree) {
  auto& t = topology(edge_type);
  const int64_t n_dst = nodes_.at(t.dst_type).num_nodes;
  auto shard_off = at::zeros({2}, at::TensorOptions().dtype(at::kLong).device(device_));   // one shard: [0, n_dst)
  shard_off.slice(0, 1).fill_(n_dst);
  c10::optional<at::Tensor> cum;
  if (by_in_degree) cum = at::bincount(t.indices, {}, n_dst).to(at::kDouble).cumsum(0).contiguous();
  return glb::negative_sample(t.desc, ids.to(device_, at::kLong), k, cum, shard_off, n_dst, strict, /*retry=*/3, /*scan_cap=*/512, rng_,
                              ++salt_, c10::nullopt);
}

Stats Graph::GetStats() const {
  Stats s;
  for (auto& kv : nodes_) s.node_count[kv.first] = kv.second.num_nodes;
  for (auto& kv : topo_) s.edge_count[kv.first] = kv.second.num_edges;
  return s;
}

// ------------------------------------------------------------------------------------------------ Query
Query Query::V(const std::string& node_type, const std::string& alias) {
  Query q;
  q.node_type = node_type;
  q.root_alias = alias;
  return q;
}
Query& Query::Batch(int64_t b) { batch_size = b; return *this; }
Query& Query::Shuffle(bool traverse) { shuffle = traverse; return *this; }
Query& Query::OutV(const std::string& edge_type, int64_t k, Strategy s, const std::string& alias) {
  hops.push_back(Hop{edge_type, k, s, alias});
  return *this;
}
Query& Query::WithFeatures(bool on) { features = on; return *this; }

// ------------------------------------------------------------------------------------------------ Dataset
struct Dataset::Impl {
  std::shared_ptr<Graph> g;
  Query q;
  int64_t depth;
  bool drop_last;
  int64_t n_nodes = 0, cursor = 0, produced = 0, consumed = 0;
  at::Tensor order;                      // device permutation of this epoch
  std::vector<Batch> ring;
  std::vector<at::cuda::CUDAEvent> done;
  c10::cuda::CUDAStream stream;
  bool epoch_done_producing = false;

  Impl(std::shared_ptr<Graph> g_, const Query& q_, int64_t depth_, bool drop_last_)
      : g(std::move(g_)), q(q_), depth(std::max<int64_t>(1, depth_)), drop_last(drop_last_),
        stream(c10::cuda::getStreamFromPool(false, g->device().index())) {
    n_nodes = g->nodes(q.node_type).num_nodes;
    ring.resize(depth);
    done.resize(depth);
    // the ring owns its hop buffers: sampling writes in place, nothing is allocated per batch
    auto opt = at::TensorOptions().dtype(at::kLong).device(g->device());
    for (auto& b : ring) {
      int64_t n = q.batch_size;
      b.ids.push_back(at::zeros({n}, opt));
      for (auto& h : q.hops) { n *= h.k; b.ids.push_back(at::zeros({n}, opt)); }
    }
    NewEpoch();
  }

  void NewEpoch() {
    c10::cuda::CUDAStreamGuard sg(stream);
    auto opt = at::TensorOptions().dtype(at::kLong).device(g->device());
    order = q.shuffle ? at::randperm(n_nodes, opt) : at::arange(n_nodes, opt);
    cursor = 0;
    epoch_done_producing = false;
  }

  int64_t BatchesPerEpoch() const {
    return drop_last ? n_nodes / q.batch_size : (n_nodes + q.batch_size - 1) / q.batch_size;
  }

  // enqueue the sampling of one batch into ring slot (produced % depth) on the side stream
  bool Produce() {
    if (epoch_done_producing) return false;
    const int64_t B = q.batch_size;
    int64_t m = std::min(B, n_nodes - cursor);
    if (m <= 0 || (drop_last && m < B)) { epoch_done_producing = true; return false; }
    Batch& b = ring[produced % depth];
    c10::cuda::CUDAStreamGuard sg(stream);
    b.size = m;
    b.ids[0].slice(0, 0, m).copy_(order.slice(0, cursor, cursor + m));
    if (m < B) b.ids[0].slice(0, m).fill_(-1);             // invalid ids: the samplers emit the default neighbour
    cursor += m;
    for (size_t i = 0; i < q.hops.size(); ++i) {
      const Hop& h = q.hops[i];
      g->SampleNeighbors(h.edge_type, b.ids[i], h.k, h.strategy, b.ids[i + 1], /*default_id=*/-1);
    }
    g->AdvanceRng();
    b.features.clear();
    if (q.features) {
      const std::string* type = &q.node_type;
      for (size_t i = 0; i < b.ids.size(); ++i) {
        if (i > 0) type = &g->topology(q.hops[i - 1].edge_type).dst_type;
        b.features.push_back(g->nodes(*type).features.defined() ? g->LookupNodes(*type, b.ids[i]) : at::Tensor());
      }
    }
    const auto& root = g->nodes(q.node_type);
    b.labels = root.labels.defined() ? g->LookupLabels(q.node_type, b.ids[0]) : at::Tensor();
    done[produced % depth].record(stream);
    ++produced;
    return true;
  }
};

Dataset::Dataset(std::shared_ptr<Graph> g, const Query& q, int64_t prefetch, bool drop_last) {
  TORCH_CHECK(g && g->initialized(), "Dataset needs an initialised Graph");
  TORCH_CHECK(q.batch_size > 0, "Query::Batch must be positive");
  c10::cuda::CUDAGuard guard(g->device());
  impl_ = std::make_unique<Impl>(std::move(g), q, prefetch, drop_last);
}

Dataset::~Dataset() = default;

int64_t Dataset::batches_per_epoch() const { return impl_->BatchesPerEpoch(); }

bool Dataset::Next(Batch* out) {
  Impl& d = *impl_;
  c10::cuda::CUDAGuard guard(d.g->device());
  auto cur = c10::cuda::getCurrentCUDAStream(d.g->device().index());
  // the producer must not overwrite a slot the consumer stream may still be reading
  at::cuda::CUDAEvent consumer_here;
  consumer_here.record(cur);
  consumer_here.block(d.stream);
  while (d.produced - d.consumed < d.depth && d.Produce()) {}
  if (d.produced == d.consumed) {       // epoch exhausted (the reference answers OutOfRange): rewind for the next pass
    ++epoch_;
    d.NewEpoch();
    return false;
  }
  const int64_t slot = d.consumed % d.depth;
  d.done[slot].block(cur);
  *out = d.ring[slot];
  ++d.consumed;
  return true;
}

}  // namespace api
}  // namespace glb
