// pybind11 surface of the native extension `graphlearn_b200._C`.
#include <torch/extension.h>

#include "glb/api.h"

namespace glb {
// sampling.cu
std::vector<at::Tensor> sample_neighbors(const at::Tensor&, const at::Tensor&, int64_t, int64_t, int64_t,
                                         const c10::optional<at::Tensor>&, bool, int64_t, int64_t,
                                         const at::Tensor&, int64_t, bool, const c10::optional<at::Tensor>&);
at::Tensor get_degrees(const at::Tensor&, const at::Tensor&, int64_t);
std::vector<at::Tensor> sample_full(const at::Tensor&, const at::Tensor&, int64_t, bool, int64_t);
void rng_advance(const at::Tensor&, int64_t);
// walk.cu
at::Tensor random_walk(const at::Tensor&, const at::Tensor&, int64_t, double, double, int64_t, int64_t,
                       const at::Tensor&, int64_t);
// negative.cu
at::Tensor negative_sample(const at::Tensor&, const at::Tensor&, int64_t, const c10::optional<at::Tensor>&,
                           const at::Tensor&, int64_t, bool, int64_t, int64_t, const at::Tensor&, int64_t,
                           const c10::optional<at::Tensor>&);
// gather.cu
at::Tensor gather_rows(const at::Tensor&, const at::Tensor&, bool, double);
at::Tensor gather_agg(const at::Tensor&, const at::Tensor&, const c10::optional<at::Tensor>&, int64_t, int64_t);
void scatter_add_rows(const at::Tensor&, const at::Tensor&, const at::Tensor&, double);
void sparse_adam_rows(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, double, double, double,
                      double, int64_t);
void gather_copy16(const at::Tensor&, const at::Tensor&, int64_t, const at::Tensor&, bool, int64_t);
// sage_fused.cu
int64_t sage_smem_bytes(int64_t, int64_t);
std::vector<at::Tensor> sage_fused_forward(const at::Tensor&, const c10::optional<at::Tensor>&, const at::Tensor&,
                                           const c10::optional<at::Tensor>&, int64_t, int64_t, int64_t,
                                           const at::Tensor&, const c10::optional<at::Tensor>&, int64_t, int64_t,
                                           bool, bool, bool);
void sage_fused_multi(const at::Tensor&, const at::Tensor&, const std::vector<c10::optional<at::Tensor>>&,
                      const std::vector<c10::optional<at::Tensor>>&, const std::vector<int64_t>&, const std::vector<int64_t>&,
                      const std::vector<int64_t>&, const std::vector<int64_t>&, const std::vector<at::Tensor>&,
                      const std::vector<c10::optional<at::Tensor>>&, int64_t, const at::Tensor&,
                      const c10::optional<at::Tensor>&, int64_t, int64_t, bool, bool,
                      const std::vector<c10::optional<at::Tensor>>&, int64_t, int64_t,
                      const std::vector<c10::optional<at::Tensor>>&, const c10::optional<at::Tensor>&, double, int64_t,
                      const std::vector<int64_t>&, int64_t, const std::vector<c10::optional<at::Tensor>>&);
void sage_fused_csr(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
                    const std::vector<at::Tensor>&, const at::Tensor&, int64_t, const at::Tensor&,
                    const c10::optional<at::Tensor>&, int64_t, int64_t, bool, bool, int64_t, int64_t, int64_t,
                    const c10::optional<at::Tensor>&);
int sm_count();
void sage_set_debug_trace(const c10::optional<at::Tensor>&);
// sage_bwd.cu
void sage_bwd_da(const at::Tensor&, const at::Tensor&, int64_t, int64_t, const at::Tensor&, double,
                 const std::vector<std::pair<int64_t, int64_t>>&);
void sage_bwd_dw(const c10::optional<at::Tensor>&, const c10::optional<at::Tensor>&, const std::vector<int64_t>&,
                 const std::vector<int64_t>&, const std::vector<c10::optional<at::Tensor>>&,
                 const std::vector<c10::optional<at::Tensor>>&, const std::vector<int64_t>&, const std::vector<double>&, int64_t,
                 const c10::optional<at::Tensor>&, const c10::optional<at::Tensor>&, const c10::optional<at::Tensor>&,
                 const c10::optional<at::Tensor>&, int64_t, const std::vector<double>&, const std::vector<c10::optional<at::Tensor>>&);
// sage_bn.cu
void bn_fwd_stats(const at::Tensor&, int64_t, const std::vector<int64_t>&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
                  const at::Tensor&, const at::Tensor&, const at::Tensor&, double, double);
void bn_fwd_apply(const at::Tensor&, int64_t, const std::vector<int64_t>&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
                  const at::Tensor&, const at::Tensor&, const c10::optional<at::Tensor>&, double, int64_t);
void bn_bwd_reduce(const at::Tensor&, const at::Tensor&, int64_t, const std::vector<int64_t>&, const at::Tensor&, const at::Tensor&,
                   const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&);
void bn_bwd_apply(const at::Tensor&, const at::Tensor&, int64_t, const std::vector<int64_t>&, const at::Tensor&, const at::Tensor&,
                  const at::Tensor&, const at::Tensor&, const at::Tensor&);
// sage_embed.cu
void embed_grad_scatter(const at::Tensor&, const std::vector<int64_t>&, const std::vector<at::Tensor>&, const std::vector<at::Tensor>&,
                        const std::vector<int64_t>&, const std::vector<double>&, const std::vector<double>&, int64_t,
                        const std::vector<c10::optional<at::Tensor>>&, const at::Tensor&, const at::Tensor&);
void embed_lazy_adam(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
                     const at::Tensor&, const at::Tensor&, double, double, double, double);
// train_ops.cu
void softmax_ce(const at::Tensor&, const at::Tensor&, const c10::optional<at::Tensor>&, int64_t, const at::Tensor&,
                const at::Tensor&, const c10::optional<at::Tensor>&);
void link_loss(const at::Tensor&, int64_t, int64_t, int64_t, double, const at::Tensor&, const at::Tensor&,
               const c10::optional<at::Tensor>&);
void link_roots(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, int64_t, int64_t);
std::vector<at::Tensor> pack_weight_f32(const at::Tensor&, int64_t, bool);
at::Tensor tc_linear_forward(const at::Tensor&, const at::Tensor&, const c10::optional<at::Tensor>&, int64_t, int64_t, bool,
                             bool);
// comm.cu
int64_t symm_alloc(int64_t, int64_t);
void symm_free(int64_t, int64_t);
py::bytes ipc_get_handle(int64_t, int64_t);
int64_t ipc_open_handle(const std::string&, int64_t);
void ipc_close_handle(int64_t, int64_t);
at::Tensor tensor_from_ptr(int64_t, std::vector<int64_t>, int64_t, int64_t);
void allreduce_oneshot(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, double);
void copy_i64(const at::Tensor&, const at::Tensor&);
void step_advance(const c10::optional<at::Tensor>&, const c10::optional<at::Tensor>&, int64_t);
void adam_flat(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
               double, double, double, double, double);
void adam_pack(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, double, double, double,
               double, double, const c10::optional<at::Tensor>&, const at::Tensor&, const c10::optional<at::Tensor>&,
               const c10::optional<at::Tensor>&, const c10::optional<at::Tensor>&, double, bool, const c10::optional<at::Tensor>&);
// graph_ops.cu
std::vector<at::Tensor> relabel(const at::Tensor&, bool);
at::Tensor relabel_lookup(const at::Tensor&, const at::Tensor&, const at::Tensor&);
at::Tensor edge_scatter(const at::Tensor&, const at::Tensor&, const at::Tensor&, const c10::optional<at::Tensor>&,
                        int64_t, int64_t);
at::Tensor edge_dot(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, int64_t);
// gat.cu
std::vector<at::Tensor> gat_agg_forward(const at::Tensor&, const c10::optional<at::Tensor>&, int64_t, const at::Tensor&,
                                        const c10::optional<at::Tensor>&, int64_t, int64_t, int64_t, const at::Tensor&, const at::Tensor&,
                                        const at::Tensor&, double);
std::vector<at::Tensor> gat_agg_backward(const at::Tensor&, const at::Tensor&, const c10::optional<at::Tensor>&, int64_t, int64_t, int64_t,
                                         const at::Tensor&, const at::Tensor&, const at::Tensor&, double, const at::Tensor&, const at::Tensor&,
                                         const at::Tensor&, bool);
// idmap.cu
at::Tensor idmap_translate(const at::Tensor&, const at::Tensor&, bool);
// csr_build.cu
std::vector<at::Tensor> csr_build(const at::Tensor&, int64_t, const c10::optional<at::Tensor>&, int64_t);
// knn.cu
std::vector<at::Tensor> knn_flat_topk(const at::Tensor&, int64_t, const c10::optional<at::Tensor>&, const c10::optional<at::Tensor>&,
                                      const at::Tensor&, int64_t, int64_t);
std::vector<at::Tensor> knn_ivf_search(const at::Tensor&, int64_t, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, int64_t,
                                       int64_t);
std::vector<at::Tensor> knn_merge_peers(const at::Tensor&, int64_t, int64_t, int64_t, const at::Tensor&);
std::vector<at::Tensor> knn_ivfpq_search(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
                                         const at::Tensor&, int64_t, int64_t);
// dgs.cu
void dgs_apply_edges(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&,
                     const at::Tensor&, const c10::optional<at::Tensor>&);
std::vector<at::Tensor> dgs_lookup(const at::Tensor&, const at::Tensor&, const at::Tensor&, const at::Tensor&, int64_t);
// host_loader.cpp
std::vector<at::Tensor> parse_records(const std::string&, int64_t, int64_t, const std::string&, const std::string&, const std::vector<std::string>&,
                                      const std::vector<int64_t>&, const std::vector<int64_t>&, const std::vector<int64_t>&,
                                      const std::vector<int64_t>&, const std::vector<int64_t>&, const std::vector<int64_t>&,
                                      const std::vector<int64_t>&, int64_t);
std::vector<at::Tensor> load_table(const std::string&, bool, bool, bool, bool, std::vector<int64_t>,
                                   std::vector<int64_t>, const std::string&, const std::string&, int64_t,
                                   int64_t, int64_t);
void save_embeddings(const std::string&, const at::Tensor&, const at::Tensor&, bool);
}  // namespace glb

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "graphlearn_b200 native runtime: sm_90a kernels + host loader";
  // ---- public C++ API (include/glb/api.h), exported 1:1 so the test-suite can hold it against the Python path
  {
    namespace A = glb::api;
    py::class_<A::Graph, std::shared_ptr<A::Graph>>(m, "CppGraph")
        .def(py::init<int, int64_t>(), py::arg("device_index") = 0, py::arg("seed") = 0)
        .def("add_nodes", [](A::Graph& g, const std::string& t, int64_t n, const c10::optional<at::Tensor>& f,
                             const c10::optional<at::Tensor>& l, const c10::optional<at::Tensor>& w, bool bf16) { g.AddNodes(t, n, f, l, w, bf16); },
             py::arg("type"), py::arg("num_nodes"), py::arg("features") = py::none(), py::arg("labels") = py::none(),
             py::arg("weights") = py::none(), py::arg("store_bf16") = false)
        .def("add_edges", [](A::Graph& g, const std::string& t, const std::string& s, const std::string& d, const at::Tensor& src,
                             const at::Tensor& dst, const c10::optional<at::Tensor>& w) { g.AddEdges(t, s, d, src, dst, w); },
             py::arg("type"), py::arg("src_type"), py::arg("dst_type"), py::arg("src"), py::arg("dst"), py::arg("weights") = py::none())
        .def("add_node_file", [](A::Graph& g, const std::string& t, const std::string& p, int64_t fd, bool w, bool l, bool bf16) {
          g.AddNodeFile(t, p, fd, w, l, bf16); }, py::arg("type"), py::arg("path"), py::arg("float_dim"), py::arg("weighted") = false,
             py::arg("labeled") = false, py::arg("store_bf16") = false)
        .def("add_edge_file", [](A::Graph& g, const std::string& t, const std::string& s, const std::string& d, const std::string& p, bool w) {
          g.AddEdgeFile(t, s, d, p, w); }, py::arg("type"), py::arg("src_type"), py::arg("dst_type"), py::arg("path"), py::arg("weighted") = false)
        .def("init", &A::Graph::Init)
        .def("sample_neighbors", [](A::Graph& g, const std::string& e, const at::Tensor& ids, int64_t k, const std::string& s) {
          return g.SampleNeighbors(e, ids, k, A::strategy_from_name(s)); }, py::arg("edge_type"), py::arg("ids"), py::arg("k"),
             py::arg("strategy") = "random")
        .def("full_neighbors", &A::Graph::FullNeighbors)
        .def("get_degree", &A::Graph::GetDegree)
        .def("lookup_nodes", &A::Graph::LookupNodes, py::arg("node_type"), py::arg("ids"), py::arg("out_bf16") = false)
        .def("lookup_labels", &A::Graph::LookupLabels)
        .def("random_walk", &A::Graph::RandomWalk, py::arg("edge_type"), py::arg("ids"), py::arg("walk_len"), py::arg("p") = 1.0,
             py::arg("q") = 1.0)
        .def("negative_sample", &A::Graph::NegativeSample, py::arg("edge_type"), py::arg("ids"), py::arg("k"), py::arg("strict") = true,
             py::arg("by_in_degree") = false)
        .def("get_stats", [](const A::Graph& g) { auto s = g.GetStats(); return py::make_tuple(s.node_count, s.edge_count); });
    py::class_<A::Query>(m, "CppQuery")
        .def_static("V", &A::Query::V, py::arg("node_type"), py::arg("alias") = "src")
        .def("batch", [](A::Query& q, int64_t b) { return q.Batch(b); })
        .def("shuffle", [](A::Query& q, bool t) { return q.Shuffle(t); }, py::arg("traverse") = true)
        .def("outV", [](A::Query& q, const std::string& e, int64_t k, const std::string& s, const std::string& a) {
          return q.OutV(e, k, A::strategy_from_name(s), a); }, py::arg("edge_type"), py::arg("k"), py::arg("strategy") = "random",
             py::arg("alias") = "")
        .def("with_features", [](A::Query& q, bool on) { return q.WithFeatures(on); }, py::arg("on") = true);
    py::class_<A::Dataset>(m, "CppDataset")
        .def(py::init<std::shared_ptr<A::Graph>, const A::Query&, int64_t, bool>(), py::arg("graph"), py::arg("query"),
             py::arg("prefetch") = 2, py::arg("drop_last") = false)
        .def("next", [](A::Dataset& d) -> py::object {
          A::Batch b;
          if (!d.Next(&b)) return py::none();
          return py::make_tuple(b.size, b.ids, b.features, b.labels.defined() ? py::cast(b.labels) : py::none());
        })
        .def_property_readonly("epoch", &A::Dataset::epoch)
        .def_property_readonly("batches_per_epoch", &A::Dataset::batches_per_epoch);
  }
  m.def("sample_neighbors", &glb::sample_neighbors);
  m.def("get_degrees", &glb::get_degrees);
  m.def("sample_full", &glb::sample_full);
  m.def("rng_advance", &glb::rng_advance);
  m.def("random_walk", &glb::random_walk);
  m.def("negative_sample", &glb::negative_sample);
  m.def("gather_rows", &glb::gather_rows);
  m.def("gather_agg", &glb::gather_agg);
  m.def("scatter_add_rows", &glb::scatter_add_rows);
  m.def("gather_copy16", &glb::gather_copy16);
  m.def("sparse_adam_rows", &glb::sparse_adam_rows);
  m.def("sage_smem_bytes", &glb::sage_smem_bytes);
  m.def("sage_fused_forward", &glb::sage_fused_forward);
  // (amax: per-segment argmax outputs of a max-aggregating launch, see sage_fused.cu)
  m.def("sage_fused_multi", &glb::sage_fused_multi, py::arg("tself_desc"), py::arg("tnbr_desc"), py::arg("self_vids"),
        py::arg("nbr_vids"), py::arg("self_base"), py::arg("nbr_base"), py::arg("Ms"), py::arg("ks"), py::arg("outs"),
        py::arg("a_saves"), py::arg("mode"), py::arg("w_img"), py::arg("bias"), py::arg("N"), py::arg("n_out"), py::arg("relu"),
        py::arg("out_bf16"), py::arg("ce"), py::arg("ce_world"), py::arg("n_imgs"),
        py::arg("amax") = std::vector<c10::optional<at::Tensor>>(), py::arg("drop_state") = py::none(), py::arg("drop_p") = 0.0,
        py::arg("drop_layer") = 0, py::arg("drop_row0") = std::vector<int64_t>(), py::arg("split_half") = 0,
        py::arg("partial") = std::vector<c10::optional<at::Tensor>>());
  // (split_half / partial: one half of a split-K layer, see sage_fused.cu)
  m.def("sage_fused_csr", &glb::sage_fused_csr, py::arg("tself_desc"), py::arg("tnbr_desc"), py::arg("self_vids"),
        py::arg("csr_indptr"), py::arg("csr_indices"), py::arg("hubs"), py::arg("out"), py::arg("mode"), py::arg("w_img"),
        py::arg("bias"), py::arg("N"), py::arg("n_out"), py::arg("relu"), py::arg("out_bf16"), py::arg("n_imgs"),
        py::arg("plan_deg"), py::arg("split_half") = 0, py::arg("partial") = py::none());
  m.def("sm_count", &glb::sm_count);
  m.def("sage_set_debug_trace", &glb::sage_set_debug_trace);
  // (seg_self_scale / amax_src: the gradient routing of a gcn / max aggregation above, see sage_bwd.cu)
  m.def("sage_bwd_dw", &glb::sage_bwd_dw, py::arg("dz"), py::arg("h"), py::arg("seg_row0"), py::arg("seg_row1"),
        py::arg("self_src"), py::arg("nbr_src"), py::arg("seg_k"), py::arg("seg_scale"), py::arg("nbr_col0"), py::arg("dz_out"),
        py::arg("a"), py::arg("dw"), py::arg("dbias"), py::arg("n_out"), py::arg("seg_self_scale") = std::vector<double>(),
        py::arg("amax_src") = std::vector<c10::optional<at::Tensor>>());
  // (alpha: scale of the fp32 accumulators before the bf16 store, 1 / (1 - p) below a dropout layer; kb_ranges: at most
  // two [lo, hi) ranges of 64-column blocks of da to compute, empty = all)
  m.def("sage_bwd_da", &glb::sage_bwd_da, py::arg("dz"), py::arg("w_img"), py::arg("N"), py::arg("n_imgs"), py::arg("da"),
        py::arg("alpha") = 1.0, py::arg("kb_ranges") = std::vector<std::pair<int64_t, int64_t>>());
  // batch norm of a hidden layer's segments (offs: the nseg + 1 row offsets), see sage_bn.cu
  m.def("bn_fwd_stats", &glb::bn_fwd_stats, py::arg("z"), py::arg("C"), py::arg("offs"), py::arg("ticket"), py::arg("mean"),
        py::arg("rstd"), py::arg("running_mean"), py::arg("running_var"), py::arg("num_batches_tracked"), py::arg("eps"),
        py::arg("momentum"));
  m.def("bn_fwd_apply", &glb::bn_fwd_apply, py::arg("z"), py::arg("C"), py::arg("offs"), py::arg("mean"), py::arg("rstd"),
        py::arg("gamma"), py::arg("beta"), py::arg("h"), py::arg("drop_state") = py::none(), py::arg("drop_p") = 0.0,
        py::arg("drop_layer") = 0);
  m.def("bn_bwd_reduce", &glb::bn_bwd_reduce, py::arg("dy"), py::arg("z"), py::arg("C"), py::arg("offs"), py::arg("ticket"),
        py::arg("mean"), py::arg("rstd"), py::arg("gsum"), py::arg("dgamma"), py::arg("dbeta"));
  m.def("bn_bwd_apply", &glb::bn_bwd_apply, py::arg("dy"), py::arg("z"), py::arg("C"), py::arg("offs"), py::arg("mean"),
        py::arg("rstd"), py::arg("gamma"), py::arg("gsum"), py::arg("dz"));
  m.def("embed_grad_scatter", &glb::embed_grad_scatter, py::arg("da"), py::arg("seg_row0"), py::arg("self_ids"),
        py::arg("nbr_ids"), py::arg("seg_k"), py::arg("self_scale"), py::arg("nbr_scale"), py::arg("nbr_col0"), py::arg("amax"),
        py::arg("grad"), py::arg("bits"));
  m.def("embed_lazy_adam", &glb::embed_lazy_adam, py::arg("w"), py::arg("m"), py::arg("v"), py::arg("grad"), py::arg("img"),
        py::arg("bits"), py::arg("step"), py::arg("lr"), py::arg("beta1"), py::arg("beta2"), py::arg("eps"));
  m.def("pack_weight_f32", &glb::pack_weight_f32);
  m.def("tc_linear_forward", &glb::tc_linear_forward);
  m.def("softmax_ce", &glb::softmax_ce);
  m.def("link_loss", &glb::link_loss);
  m.def("link_roots", &glb::link_roots);
  m.def("symm_alloc", &glb::symm_alloc);
  m.def("symm_free", &glb::symm_free);
  m.def("ipc_get_handle", &glb::ipc_get_handle);
  m.def("ipc_open_handle", &glb::ipc_open_handle);
  m.def("ipc_close_handle", &glb::ipc_close_handle);
  m.def("tensor_from_ptr", &glb::tensor_from_ptr);
  m.def("allreduce_oneshot", &glb::allreduce_oneshot);
  m.def("step_advance", &glb::step_advance);
  m.def("copy_i64", &glb::copy_i64);
  m.def("adam_flat", &glb::adam_flat);
  m.def("adam_pack", &glb::adam_pack, py::arg("w"), py::arg("g_store"), py::arg("m"), py::arg("v"), py::arg("step"), py::arg("lr"),
        py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("weight_decay"), py::arg("loss_out"), py::arg("mats"),
        py::arg("ar_desc"), py::arg("ar_epochs"), py::arg("ar_error"), py::arg("ar_scale"), py::arg("stage_bf16"),
        py::arg("drop_ctr") = py::none());
  m.def("relabel", &glb::relabel);
  m.def("relabel_lookup", &glb::relabel_lookup);
  m.def("edge_scatter", &glb::edge_scatter);
  m.def("edge_dot", &glb::edge_dot);
  m.def("gat_agg_forward", &glb::gat_agg_forward);
  m.def("gat_agg_backward", &glb::gat_agg_backward);
  m.def("idmap_translate", &glb::idmap_translate);
  m.def("csr_build", &glb::csr_build);
  m.def("knn_flat_topk", &glb::knn_flat_topk);
  m.def("knn_merge_peers", &glb::knn_merge_peers);
  m.def("knn_ivf_search", &glb::knn_ivf_search);
  m.def("knn_ivfpq_search", &glb::knn_ivfpq_search);
  m.def("dgs_apply_edges", &glb::dgs_apply_edges);
  m.def("dgs_lookup", &glb::dgs_lookup);
  m.def("load_table", &glb::load_table);
  m.def("parse_records", &glb::parse_records);
  m.def("save_embeddings", &glb::save_embeddings);
}
