// Embedding graphlearn_b200 in a C++ program (public header include/glb/api.h; the reference's counterpart is a C++
// client of src/include/{client,dag_dataset}.h): build a graph from tensors, run single operators, then stream an epoch
// of a 2-hop GSL-style query through the prefetching Dataset.
//
// Build:  make -C examples/cpp        (after `python -m graphlearn_b200._build`; links _C.so + libtorch + libpython)
// Run on a machine with an H100:  ./sample_and_lookup
#include <cstdio>
#include <memory>

#include <ATen/ATen.h>

#include "glb/api.h"

int main() {
  using namespace glb::api;
  const int64_t n = 10000, deg = 8, dim = 32;
  auto dev = at::Device(at::kCUDA, 0);
  auto opt_i = at::TensorOptions().dtype(at::kLong).device(dev);
  auto opt_f = at::TensorOptions().dtype(at::kFloat).device(dev);

  // a ring-with-chords graph: i -> (i + 1 .. i + deg) mod n, heavier weights on nearer neighbours
  auto src = at::arange(n, opt_i).repeat_interleave(deg);
  auto hop = at::arange(1, deg + 1, opt_i).repeat({n});
  auto dst = (src + hop).remainder(n);
  auto w = 1.0 / hop.to(at::kFloat);
  auto feats = at::arange(n, opt_f).unsqueeze(1).expand({n, dim}).contiguous();      // feature row i == i
  auto labels = at::arange(n, opt_i).remainder(7);

  auto g = std::make_shared<Graph>(/*device_index=*/0, /*seed=*/42);
  g->AddNodes("item", n, feats, labels).AddEdges("sim", "item", "item", src, dst, w);
  g->Init();
  Stats st = g->GetStats();
  std::printf("nodes %lld edges %lld\n", (long long)st.node_count["item"], (long long)st.edge_count["sim"]);

  auto seeds = at::arange(5, opt_i);
  auto top = g->SampleNeighbors("sim", seeds, 3, Strategy::kTopK).cpu();             // the three heaviest edges: +1, +2, +3
  bool ok = true;
  for (int64_t i = 0; i < 5; ++i)
    for (int64_t j = 0; j < 3; ++j) ok = ok && top[i][j].item<int64_t>() == (i + j + 1) % n;
  auto rnd = g->SampleNeighbors("sim", seeds, 4, Strategy::kRandom).cpu();
  auto delta = (rnd - seeds.cpu().unsqueeze(1)).remainder(n);
  ok = ok && delta.ge(1).all().item<bool>() && delta.le(deg).all().item<bool>();
  ok = ok && g->GetDegree("sim", seeds).cpu().eq(deg).all().item<bool>();
  auto rows = g->LookupNodes("item", seeds).cpu();
  ok = ok && rows.select(1, 0).eq(at::arange(5, at::kFloat)).all().item<bool>();
  auto walks = g->RandomWalk("sim", seeds, 6).cpu();
  ok = ok && walks.size(0) == 5 && walks.size(1) == 6;
  std::printf("operators %s\n", ok ? "ok" : "WRONG");

  // one epoch of V("item").batch(512).shuffle().outV("sim").sample(5).outV("sim").sample(3).values()
  Query q = Query::V("item").Batch(512).Shuffle(true).OutV("sim", 5).OutV("sim", 3).WithFeatures(true);
  Dataset ds(g, q, /*prefetch=*/3);
  Batch b;
  int64_t seen = 0, batches = 0;
  while (ds.Next(&b)) {
    seen += b.size;
    ++batches;
    ok = ok && b.ids[1].numel() == b.ids[0].numel() * 5 && b.ids[2].numel() == b.ids[1].numel() * 3 &&
         b.features[2].size(1) == dim;
  }
  std::printf("epoch: %lld seeds in %lld batches (%lld expected) %s\n", (long long)seen, (long long)batches,
              (long long)ds.batches_per_epoch(), ok && seen == n ? "ok" : "WRONG");
  return ok && seen == n ? 0 : 1;
}
