"""Streaming sampler service (GPU-native DGS analogue) - semantics vs a Python oracle."""
import numpy as np
import pytest
import torch

from graphlearn_b200.dgs import AdaptiveRateLimiter, DynamicGraphService, QueryPlan


def test_topk_by_timestamp_streaming():
    schema = {"vertices": {"u": {"count": 20, "feat_dim": 3}, "i": {"count": 30, "feat_dim": 2}},
              "edges": {"click": {"src": "u", "dst": "i"}, "sim": {"src": "i", "dst": "i"}}}
    svc = DynamicGraphService(schema, device="cpu")
    svc.install_query(1, QueryPlan("u").out("click", 4).out("sim", 2))
    rs = np.random.RandomState(0)
    oracle = {}
    t = 0
    for b in range(6):
        n = 200
        src, dst = rs.randint(0, 20, n), rs.randint(0, 30, n)
        ts = np.arange(t, t + n); t += n
        svc.apply_updates({"edges": {"click": {"src": src, "dst": dst, "ts": ts}}})
        for s, d, x in zip(src, dst, ts):
            oracle.setdefault(int(s), []).append((int(x), int(d)))
    res = svc.run_query(1, list(range(20)))
    ids, tss = res["hops"][0]["ids"], res["hops"][0]["timestamps"]
    for u in range(20):
        want = sorted(oracle[u], reverse=True)[:4]
        assert [int(x) for x in tss[u]] == [w[0] for w in want]
        assert [int(x) for x in ids[u]] == [w[1] for w in want]
    assert res["hops"][1]["ids"].shape == (80, 2) and bool((res["hops"][1]["ids"] == -1).all())   # no sim edges yet
    # vertex features: latest version wins
    svc.apply_updates({"vertices": {"i": {"id": [5, 5, 6], "ts": [1, 9, 3], "feat": [[1, 1], [2, 2], [3, 3]]}}})
    svc.apply_updates({"vertices": {"i": {"id": [5], "ts": [4], "feat": [[7, 7]]}}})
    assert svc.vstores["i"].feat[5].tolist() == [2.0, 2.0] and svc.vstores["i"].feat[6].tolist() == [3.0, 3.0]
    # checkpoint / restore
    ck = svc.checkpoint()
    svc2 = DynamicGraphService(schema, device="cpu")
    svc2.install_query(1, QueryPlan("u").out("click", 4).out("sim", 2))
    svc2.restore(ck)
    assert torch.equal(svc2.run_query(1, [3])["hops"][0]["ids"], svc.run_query(1, [3])["hops"][0]["ids"])


def test_rate_limiter():
    rl = AdaptiveRateLimiter(target_ms=20, max_concurrency=27, stable_windows=2)
    for _ in range(100):
        rl.record(50.0)
    assert rl.tick() == 9
    for w in range(2):
        for _ in range(100):
            rl.record(1.0)
        c = rl.tick()
    assert c == 11


def test_reference_config_formats_file_loader_http_and_checkpoints(tmp_path):
    """The reference's own schema / install-query JSON drive the service; records come from a pattern
    file; inference goes through the HTTP front end; a checkpoint restores into a fresh service."""
    import json
    import urllib.request
    from graphlearn_b200.dgs import (CheckpointManager, FileLoader, HttpFrontEnd, Options, QueryPlan, Schema)
    schema_json = {
        "attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}, {"type": 1, "name": "weight", "value_type": "FLOAT32"},
                      {"type": 2, "name": "feature", "value_type": "FLOAT32_LIST"}],
        "vertex_defs": [{"vtype": 0, "name": "user", "attr_types": [0, 2]}, {"vtype": 1, "name": "item", "attr_types": [0, 2]}],
        "edge_defs": [{"etype": 2, "name": "u2i", "attr_types": [0, 1]}, {"etype": 3, "name": "i2i", "attr_types": [0, 1]}],
        "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}, {"etype": 3, "src_vtype": 1, "dst_vtype": 1}]}
    sp = tmp_path / "schema.json"
    sp.write_text(json.dumps(schema_json))
    schema = Schema.from_json(str(sp))
    assert schema.relations == {"u2i": ("user", "item"), "i2i": ("item", "item")}
    (tmp_path / "opt.yml").write_text("worker-type: Serving\nrecord-polling:\n  process-concurrency: 4\n")
    opt = Options.from_yaml(str(tmp_path / "opt.yml"))
    assert opt.get("record-polling.process-concurrency") == 4 and opt.get("record-polling.retry-interval-ms") == 1000

    def node(i, kind, links, **params):
        return {"id": i, "kind": kind, "type": "EDGE" if kind == "EDGE_SAMPLER" else "VERTEX",
                "links": [{"node": l, "src_output": 0, "dst_input": 0} for l in links],
                "params": [{"key": k, "value": v} for k, v in params.items()]}
    install = {"query_id": 7, "query_plan": {"plan_nodes": [
        node(0, "SOURCE", [1, 2], vtype=0, versions=1), node(1, "VERTEX_SAMPLER", [], vtype=0, versions=1),
        node(2, "EDGE_SAMPLER", [3, 4], vtype=0, etype=2, fanout=3, strategy=0),
        node(3, "VERTEX_SAMPLER", [], vtype=1, versions=1), node(4, "EDGE_SAMPLER", [], vtype=1, etype=3, fanout=2, strategy=0)]}}
    plan = QueryPlan.from_json(install, schema)
    assert plan.hops == [("u2i", 3), ("i2i", 2)]
    svc = DynamicGraphService(schema.to_service_schema(capacity=4, feat_dims={"user": 2, "item": 2}), device="cpu")
    front = HttpFrontEnd(svc, schema, checkpoint_dir=str(tmp_path / "ck")).start()
    base = "http://127.0.0.1:%d" % front.port

    def call(path, body=None):
        req = urllib.request.Request(base + path, data=None if body is None else json.dumps(body).encode(),
                                     method="GET" if body is None else "POST")
        with urllib.request.urlopen(req, timeout=10) as r:
            return json.loads(r.read())
    try:
        assert call("/admin/init", install)["query_id"] == 7
        (tmp_path / "pattern").write_text("#VERTEX:user,vid,timestamp,feature\n#VERTEX:item,vid,timestamp,feature\n"
                                          "#EDGE:u2i,src,dst,timestamp,weight\n#EDGE:i2i,src,dst,timestamp,weight\n")
        lines = ["user,%d,1,0.5:%d" % (u, u) for u in range(10)] + ["item,%d,1,%d:0.25" % (i, i) for i in range(40)]
        want = {}
        for t in range(200):
            u, i = t % 10, (t * 7) % 40
            lines.append("u2i,%d,%d,%d,1.5" % (u, i, 100 + t))
            want.setdefault(u, []).append((100 + t, i))
            lines.append("i2i,%d,%d,%d,0.5" % (i, (i + 1) % 40, 100 + t))
        (tmp_path / "data").write_text("\n".join(lines) + "\n")
        n = FileLoader(str(tmp_path / "pattern"), schema, batch_size=64).load(str(tmp_path / "data"), svc)
        assert n == len(lines) and svc.stores["u2i"].n >= 10          # tables grew past the initial capacity 4
        res = call("/infer?qid=7&vid=3,4")
        nodes = res["nodes"]
        e = [v for v in nodes.values() if v.get("edge_type") == "u2i"][0]
        for row, u in zip(e["ids"], (3, 4)):
            assert row == [i for _, i in sorted(want[u], reverse=True)[:3]]
        e2 = [v for v in nodes.values() if v.get("edge_type") == "i2i"][0]
        assert e2["ids"][0][0] == (e["ids"][0][0] + 1) % 40
        vs = [v for v in nodes.values() if v["kind"] == "VERTEX_SAMPLER" and len(v["ids"]) == 2][0]
        assert vs["features"][0] == [0.5, 3.0]
        call("/admin/barrier/set?name=b1&produced=%d" % (svc.ingested + 5), {})
        assert call("/admin/barrier/status?name=b1")["status"] == "PRODUCED"
        call("/admin/ingest", {"edges": {"u2i": {"src": [1] * 5, "dst": [2] * 5, "ts": list(range(900, 905))}}})
        assert call("/admin/barrier/status?name=b1")["status"] == "READY"
        assert call("/admin/checkpoint", {})["checkpoint_id"] == 1
        assert call("/admin/stats")["served"] == 2
    finally:
        front.stop()
    svc2 = DynamicGraphService(schema.to_service_schema(capacity=4, feat_dims={"user": 2, "item": 2}), device="cpu")
    assert CheckpointManager(svc2, str(tmp_path / "ck")).restore_latest() == 1
    a, b = svc.run_query(7, [1, 3]), svc2.run_query(7, [1, 3])
    assert torch.equal(a["hops"][0]["ids"], b["hops"][0]["ids"]) and torch.equal(a["hops"][1]["ids"], b["hops"][1]["ids"])


def test_gsl_client_over_http(tmp_path):
    """dgs/client.py (the role of the reference's Java GSL client): fluent traversal -> install-query JSON -> /admin/init,
    run -> alias-keyed numpy results, EgoGraph hop tensors, barrier / schema / registered-query calls, error paths."""
    import numpy as np
    from graphlearn_b200.dgs import HttpFrontEnd, Schema
    from graphlearn_b200.dgs import client as C
    schema = Schema({
        "attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}, {"type": 2, "name": "feature", "value_type": "FLOAT32_LIST"}],
        "vertex_defs": [{"vtype": 0, "name": "user", "attr_types": [0, 2]}, {"vtype": 1, "name": "item", "attr_types": [0, 2]}],
        "edge_defs": [{"etype": 2, "name": "u2i", "attr_types": [0]}, {"etype": 3, "name": "i2i", "attr_types": [0]}],
        "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}, {"etype": 3, "src_vtype": 1, "dst_vtype": 1}]})
    svc = DynamicGraphService(schema.to_service_schema(capacity=64, feat_dims={"user": 2, "item": 3}), device="cpu")
    front = HttpFrontEnd(svc, schema).start()
    try:
        g = C.Graph.connect("127.0.0.1:%d" % front.port)
        assert g.get_schema()["relations"] == {"u2i": ("user", "item"), "i2i": ("item", "item")}
        with pytest.raises(C.UserException):
            g.V("nobody")
        with pytest.raises(C.UserException):
            g.V("user").outV("i2i")                      # i2i starts at items
        with pytest.raises(C.UserException):
            g.V("user").outV("u2i").sample(3).by("random")
        with pytest.raises(C.UserException):
            g.V("user").outV("u2i").sample(3).values()   # no data source
        src = C.DataSource([3, 4, 5], batch=2)
        q = (g.V("user").feed(src).properties(1).alias("seed")
              .outV("u2i").sample(3).by("topk_by_timestamp").properties(1).alias("hop1")
              .outV("i2i").sample(2).by("topk_by_timestamp").alias("hop2").values())
        kinds = [n["kind"] for n in q.to_json()["query_plan"]["plan_nodes"]]
        assert kinds == ["SOURCE", "VERTEX_SAMPLER", "EDGE_SAMPLER", "VERTEX_SAMPLER", "EDGE_SAMPLER"]
        with pytest.raises(C.UserException):
            g.run(q)                                     # not installed yet
        assert g.install_async(q).result(timeout=10).ok() and q.id is not None
        svc.apply_updates({"vertices": {"user": {"id": list(range(8)), "ts": [1] * 8, "feat": [[u, 0.5] for u in range(8)]},
                                        "item": {"id": list(range(20)), "ts": [1] * 20, "feat": [[i, 1.0, 2.0] for i in range(20)]}},
                           "edges": {"u2i": {"src": [3, 3, 3, 3, 4], "dst": [10, 11, 12, 13, 14], "ts": [5, 6, 7, 8, 9]},
                                     "i2i": {"src": [13, 13, 12], "dst": [1, 2, 3], "ts": [1, 2, 3]}}})
        v = g.run(q)                                     # ids 3, 4 from the data source
        assert v["seed"]["ids"].tolist() == [3, 4] and np.allclose(v["seed"]["features"], [[3, 0.5], [4, 0.5]])
        assert v["hop1"]["ids"].tolist() == [[13, 12, 11], [14, -1, -1]]
        assert v["hop1"]["features"].shape == (2, 3, 3) and v["hop1"]["features"][0, 0].tolist() == [13.0, 1.0, 2.0]
        assert v["hop2"]["ids"].reshape(2, 3, 2)[0].tolist() == [[2, 1], [3, -1], [-1, -1]]
        ego = v.ego_graph()
        assert ego.num_hops() == 2 and ego.fanouts == [3, 2] and ego.get_vtype(1) == 1
        xs = ego.hop_tensors()
        assert [x.shape for x in xs] == [(2, 2), (6, 3), (12, 3)] and xs[1][4].tolist() == [0, 0, 0]
        v2 = g.run_async(q).result(timeout=10)           # the last id of the source
        assert v2["seed"]["ids"].tolist() == [5] and not src.has_next()
        with pytest.raises(C.UserException):
            g.run(q)                                     # source exhausted
        assert g.run(q, [3])["hop1"]["ids"].tolist() == [[13, 12, 11]]
        back = g.get_query()
        assert back.id == q.id and back.aliases() == q.aliases()
        front.barriers.set("b", svc.ingested + 100)
        assert g.check_barrier("b").code == C.Status.NOT_READY
        front.barriers.set("b2", 0)
        assert g.check_barrier("b2").ok()
        assert g.stats()["served"] >= 4
        bad = C.Query.from_json({"query_plan": {"plan_nodes": [{"id": 0, "kind": "SOURCE", "params": [{"key": "vtype", "value": 9}]}]}})
        assert not g.install(bad).ok()
        g.close()
    finally:
        front.stop()


def test_partitioned_service_matches_single_store():
    """D1 partitioner / router: P vid-hash partitions answer exactly like one store."""
    from graphlearn_b200.dgs import PartitionedGraphService
    schema = {"vertices": {"u": {"count": 16, "feat_dim": 2}, "i": {"count": 16, "feat_dim": 3}},
              "edges": {"click": {"src": "u", "dst": "i"}, "sim": {"src": "i", "dst": "i"}}}
    one = DynamicGraphService(schema, device="cpu")
    many = PartitionedGraphService(schema, num_partitions=3, devices=["cpu"] * 3)
    plan = QueryPlan("u").out("click", 3).out("sim", 2)
    one.install_query(0, plan); many.install_query(0, plan)
    rs = np.random.RandomState(1)
    t = 0
    for _ in range(5):
        n = 150
        b = {"edges": {"click": {"src": rs.randint(0, 40, n), "dst": rs.randint(0, 50, n), "ts": np.arange(t, t + n)},
                       "sim": {"src": rs.randint(0, 50, n), "dst": rs.randint(0, 50, n), "ts": np.arange(t, t + n),
                               "weight": rs.rand(n).astype(np.float32)}},
             "vertices": {"i": {"id": rs.randint(0, 50, 20), "ts": np.arange(t, t + 20), "feat": rs.randn(20, 3).astype(np.float32)}}}
        t += n
        one.apply_updates(b); many.apply_updates(b)
    q = list(range(40)) + [45]           # 45: beyond every stored vertex
    a, c = one.run_query(0, q), many.run_query(0, q)
    for h in range(2):
        for key in ("ids", "timestamps", "weights", "features"):
            assert torch.allclose(a["hops"][h][key].float(), c["hops"][h][key].float()), (h, key)
    ck = many.checkpoint()
    again = PartitionedGraphService(schema, num_partitions=3, devices=["cpu"] * 3)
    again.install_query(0, plan); again.restore(ck)
    assert torch.equal(again.run_query(0, q)["hops"][1]["ids"], c["hops"][1]["ids"]) and many.stats()["ingested"] == one.ingested


def test_sample_ttl_and_adaptive_ingest(tmp_path):
    from graphlearn_b200.dgs import FileLoader, Schema
    schema = {"vertices": {"u": {"count": 8, "feat_dim": 0}, "i": {"count": 8, "feat_dim": 0}},
              "edges": {"click": {"src": "u", "dst": "i"}}}
    svc = DynamicGraphService(schema, device="cpu")
    svc.install_query(0, QueryPlan("u").out("click", 4))
    svc.apply_updates({"edges": {"click": {"src": [1, 1, 1, 2], "dst": [3, 4, 5, 6], "ts": [10, 20, 30, 40]}}})
    assert svc.expire(25) == 2
    r = svc.run_query(0, [1, 2])["hops"][0]
    assert r["ids"][0].tolist() == [5, -1, -1, -1] and r["ids"][1].tolist() == [6, -1, -1, -1]
    assert svc.stores["click"].count[1].item() == 1
    # adaptive ingest: slow queries shrink the ingest batch, the loader restores its nominal size afterwards
    sj = {"attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}],
          "vertex_defs": [{"vtype": 0, "name": "u", "attr_types": [0]}, {"vtype": 1, "name": "i", "attr_types": [0]}],
          "edge_defs": [{"etype": 2, "name": "click", "attr_types": [0]}],
          "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}]}
    (tmp_path / "pat").write_text("#EDGE:click,src,dst,timestamp\n")
    (tmp_path / "data").write_text("".join("click,%d,%d,%d\n" % (i % 8, (i * 3) % 8, 100 + i) for i in range(500)))
    for _ in range(50):
        svc.limiter.record(1000.0)                      # pretend the serving latency target is being missed
    fl = FileLoader(str(tmp_path / "pat"), Schema(sj), batch_size=64)
    assert fl.load(str(tmp_path / "data"), svc, adaptive=True) == 500
    assert svc.limiter.concurrency < svc.limiter.max_c and fl.batch_size == 64
    assert svc.run_query(0, [3])["hops"][0]["timestamps"][0, 0].item() == 100 + 499 - (499 - 3) % 8


def test_streaming_cluster_subscriptions_match_single_store(tmp_path):
    """D5/D7/D8/D9/D12: sampling workers publish only subscribed rows, serving workers answer from local caches exactly
    like the monolithic store - also for vertices that become reachable late (rule back-fill) - and a coordinator
    checkpoint + channel replay restores the whole pipeline."""
    from graphlearn_b200.dgs import Coordinator, PlanNode, StreamingCluster
    schema = {"vertices": {"u": {"count": 16, "feat_dim": 0}, "i": {"count": 16, "feat_dim": 3}},
              "edges": {"click": {"src": "u", "dst": "i"}, "sim": {"src": "i", "dst": "i"}}}
    plan = QueryPlan("u").out("click", 3).out("sim", 2)
    plan.add(PlanNode(3, "VERTEX_SAMPLER", vtype="i", parent=1))          # features of the 1-hop items
    one = DynamicGraphService(schema, device="cpu")
    one.install_query(0, plan)
    cl = StreamingCluster(schema, num_sampling=3, num_serving=2, sampling_devices=["cpu"] * 3, serving_devices=["cpu"] * 2,
                          log_dir=str(tmp_path / "logs"))
    cl.install_query(plan)
    co = Coordinator(cl, meta_dir=str(tmp_path / "meta"))
    info = co.register_worker("sampling", 0, "127.0.0.1:1")
    assert info["num_serving"] == 2 and info["query_plan"]["source"] == "u" and not co.ready()
    for k, n in (("sampling", 3), ("serving", 2)):
        for w in range(n):
            co.register_worker(k, w); co.report_started(k, w)
    assert co.ready() and co.sampling.all_registered()
    co.register_worker("sampling", 1)                                     # a restart resets the dependent group
    assert not co.sampling.all_registered() and co.serving.all_started()

    rs = np.random.RandomState(3)
    t = 0

    def batch(n=120):
        nonlocal t
        b = {"edges": {"sim": {"src": rs.randint(0, 50, n), "dst": rs.randint(0, 50, n), "ts": np.arange(t, t + n),
                               "weight": rs.rand(n).astype(np.float32)},
                       "click": {"src": rs.randint(0, 40, n), "dst": rs.randint(0, 50, n), "ts": np.arange(t, t + n)}},
             "vertices": {"i": {"id": rs.randint(0, 50, 20), "ts": np.arange(t, t + 20), "feat": rs.randn(20, 3).astype(np.float32)}}}
        t += n
        return b

    def same(q):
        a, c = one.run_query(0, q), cl.run_query(q)
        for h in range(2):
            for key in ("ids", "timestamps", "weights"):
                assert torch.allclose(a["hops"][h][key].float(), c["hops"][h][key].float()), (h, key)
        assert torch.allclose(a["nodes"][3]["features"], c["nodes"][3]["features"])

    q = list(range(40)) + [45]
    for r in range(4):
        b = batch()
        one.apply_updates(b)
        assert cl.produce(b) == 260
        if r == 1:
            co.set_barrier("b")
            assert co.barrier_status("b") == "PRODUCED"
        cl.pump()
        if r == 1:
            assert co.barrier_status("b") == "READY" and cl.barrier_ready()
        same(q)
    st = cl.stats()
    total_rows = sum(s["published_rows"] for s in st["sampling"])
    assert st["produced"] == 4 * 260 and sum(s["applied"] for s in st["sampling"]) == 4 * 260 and total_rows > 0
    # a serving worker only ever receives the "sim" rows of items it subscribed to (reachable from one of ITS users)
    for w in cl.serving:
        have = set((w.rows[2]["nbr"][:, 0] >= 0).nonzero().flatten().tolist())
        subscribed = set()
        for sw in cl.sampling:
            m = sw.subs.mask[2]
            subscribed |= set((((m >> w.wid) & 1) == 1).nonzero().flatten().tolist())
        assert have <= subscribed and len(subscribed) > 0

    cid = co.checkpoint()
    assert cid == 1 and co.latest_checkpoint() == 1
    more = batch()
    one.apply_updates(more); cl.produce(more)                              # produced AFTER the checkpoint, not yet consumed
    cl2 = StreamingCluster(schema, num_sampling=3, num_serving=2, sampling_devices=["cpu"] * 3, serving_devices=["cpu"] * 2,
                           log_dir=str(tmp_path / "logs"))                 # recovers the channel segments from disk
    co2 = Coordinator(cl2, meta_dir=str(tmp_path / "meta"))
    assert co2.restore_latest() == 1
    cl2.pump()                                                             # replays the batch from the checkpointed offsets
    a, c = one.run_query(0, q), cl2.run_query(q)
    assert torch.equal(a["hops"][1]["ids"], c["hops"][1]["ids"]) and torch.equal(a["hops"][0]["ids"], c["hops"][0]["ids"])


def test_group_producer_sdk(tmp_path):
    """D13 data-loader SDK: per-partition batching into the cluster's ingest log + barrier through the coordinator"""
    from graphlearn_b200.dgs import Coordinator, GroupProducer, StreamingCluster
    schema = {"vertices": {"u": {"count": 8, "feat_dim": 0}, "i": {"count": 8, "feat_dim": 2}},
              "edges": {"click": {"src": "u", "dst": "i"}}}
    plan = QueryPlan("u").out("click", 2)
    cl = StreamingCluster(schema, num_sampling=2, num_serving=1, sampling_devices=["cpu"] * 2, serving_devices=["cpu"])
    cl.install_query(plan)
    co = Coordinator(cl)
    one = DynamicGraphService(schema, device="cpu")
    one.install_query(0, plan)
    gp = GroupProducer(cl, max_batch_size=5)
    ref = GroupProducer(one, max_batch_size=1000, num_partitions=1)
    rs = np.random.RandomState(0)
    for t in range(37):
        s, d = int(rs.randint(0, 12)), int(rs.randint(0, 9))
        gp.add_edge("click", s, d, t); ref.add_edge("click", s, d, t)
    assert cl.ingest.end_offset(0) + cl.ingest.end_offset(1) >= 6          # full batches were produced on the fly
    gp.set_barrier(co, "all")
    ref.flush_all()
    assert gp.produced == 37 and cl.produced == 37 and co.barrier_status("all") == "PRODUCED"
    cl.pump()
    assert co.barrier_status("all") == "READY"
    q = list(range(12))
    a, c = one.run_query(0, q), cl.run_query(q)
    assert torch.equal(a["hops"][0]["ids"], c["hops"][0]["ids"])


def test_record_batch_wire_format_roundtrip():
    """D2: columnar binary record batches (header + raw column buffers)"""
    from graphlearn_b200.dgs import decode_record_batch, encode_record_batch
    rs = np.random.RandomState(0)
    b = {"edges": {"click": {"src": rs.randint(0, 9, 7), "dst": rs.randint(0, 9, 7), "ts": np.arange(7), "weight": rs.rand(7).astype(np.float32)},
                   "sim": {"src": torch.arange(3), "dst": torch.arange(3) + 1, "ts": torch.arange(3), "weight": None}},
         "vertices": {"i": {"id": np.arange(4), "ts": np.arange(4), "feat": rs.randn(4, 3).astype(np.float32)}}, "_n": 14}
    buf = encode_record_batch(b)
    d = decode_record_batch(buf)
    assert d["_n"] == 14 and set(d["edges"]) == {"click", "sim"} and "weight" not in d["edges"]["sim"]
    assert np.array_equal(d["edges"]["click"]["src"], b["edges"]["click"]["src"]) and d["edges"]["click"]["weight"].dtype == np.float32
    assert np.array_equal(d["edges"]["sim"]["dst"], np.arange(3) + 1)
    assert np.array_equal(d["vertices"]["i"]["feat"], b["vertices"]["i"]["feat"]) and d["vertices"]["i"]["feat"].shape == (4, 3)
    svc = DynamicGraphService({"vertices": {"u": {"count": 16, "feat_dim": 0}, "i": {"count": 16, "feat_dim": 3}},
                               "edges": {"click": {"src": "u", "dst": "i"}, "sim": {"src": "i", "dst": "i"}}}, device="cpu")
    svc.install_query(0, QueryPlan("u").out("click", 2))
    svc.apply_updates(d)                                   # decoded (read-only) views feed the service directly
    assert svc.ingested == 7
    try:
        decode_record_batch(b"nonsense")
        assert False
    except ValueError:
        pass


def test_service_process_entry_point(tmp_path):
    """``python -m graphlearn_b200.dgs`` (what the Helm chart in deploy/dgs runs): starts from schema + install-query files,
    serves, writes a final checkpoint on SIGTERM and restores it (query included) on the next start."""
    import json
    import os
    import signal
    import subprocess
    import sys
    import time
    from graphlearn_b200.dgs import client as C
    schema = {"attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}],
              "vertex_defs": [{"vtype": 0, "name": "user", "attr_types": [0]}, {"vtype": 1, "name": "item", "attr_types": [0]}],
              "edge_defs": [{"etype": 2, "name": "u2i", "attr_types": [0]}],
              "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}]}
    (tmp_path / "schema.json").write_text(json.dumps(schema))
    install = {"query_id": 3, "query_plan": {"plan_nodes": [
        {"id": 0, "kind": "SOURCE", "links": [{"node": 1}], "params": [{"key": "vtype", "value": 0}]},
        {"id": 1, "kind": "EDGE_SAMPLER", "links": [], "params": [{"key": "vtype", "value": 0}, {"key": "etype", "value": 2},
                                                                   {"key": "fanout", "value": 2}, {"key": "strategy", "value": 0}]}]}}
    (tmp_path / "q.json").write_text(json.dumps(install))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))

    def start(extra=()):
        pf = tmp_path / "port"
        if pf.exists():
            pf.unlink()
        p = subprocess.Popen([sys.executable, "-m", "graphlearn_b200.dgs", "--schema", str(tmp_path / "schema.json"), "--device", "cpu",
                              "--host", "127.0.0.1", "--port", "0", "--capacity", "16", "--checkpoint-dir", str(tmp_path / "ck"),
                              "--port-file", str(pf)] + list(extra), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        t0 = time.time()
        while not pf.exists() and time.time() - t0 < 120 and p.poll() is None:
            time.sleep(0.2)
        assert pf.exists(), p.communicate(timeout=5)[0]
        return p, int(pf.read_text())
    p, port = start(["--install-query", str(tmp_path / "q.json")])
    try:
        g = C.Graph.connect("127.0.0.1:%d" % port)
        g._http("POST", "/admin/ingest", {"edges": {"u2i": {"src": [1, 1, 1], "dst": [4, 5, 6], "ts": [10, 11, 12]}}})
        q = g.get_query(3) if False else C.Query.from_json(install)
        q.id = 3
        assert g.run(q, [1]).node(1)["ids"].tolist() == [[6, 5]]
    finally:
        p.send_signal(signal.SIGTERM)
        out = p.communicate(timeout=60)[0].decode()
    assert "final checkpoint 1" in out, out
    p, port = start()                                    # no --install-query: the checkpoint carries it
    try:
        g = C.Graph.connect("127.0.0.1:%d" % port)
        assert g.run(q, [1]).node(1)["ids"].tolist() == [[6, 5]]
        assert g.stats()["ingested"] == 3
    finally:
        p.send_signal(signal.SIGTERM)
        out = p.communicate(timeout=60)[0].decode()
    assert "restored checkpoint 1" in out, out


def test_key_level_ops_and_backup_engine(tmp_path):
    """SampleStore get / get_vertex / delete (the reference's KV surface), vertex deletion cascading to the edge stores,
    CheckpointManager as a backup engine: list, restore a chosen id (newer rows must vanish), purge."""
    from graphlearn_b200.dgs import CheckpointManager
    schema = {"vertices": {"u": {"count": 8, "feat_dim": 2}, "i": {"count": 8, "feat_dim": 0}},
              "edges": {"click": {"src": "u", "dst": "i"}}}
    svc = DynamicGraphService(schema, device="cpu")
    svc.install_query(0, QueryPlan("u").out("click", 3))
    svc.apply_updates({"vertices": {"u": {"id": [1, 2], "ts": [5, 6], "feat": [[1.0, 1.5], [2.0, 2.5]]}},
                       "edges": {"click": {"src": [1, 1, 1, 1, 2], "dst": [3, 4, 5, 6, 7], "ts": [10, 40, 20, 30, 50], "weight": [1, 2, 3, 4, 5]}}})
    st = svc.stores["click"]
    nbr, ts, w = st.get(1)
    assert nbr.tolist() == [4, 6, 5] and ts.tolist() == [40, 30, 20] and w.tolist() == [2.0, 4.0, 3.0]   # newest first, oldest evicted
    assert st.get(5)[0].numel() == 0 and st.get(10 ** 9)[0].numel() == 0
    f, fts = svc.vstores["u"].get_vertex(2)
    assert f.tolist() == [2.0, 2.5] and fts == 6 and svc.vstores["u"].get_vertex(3) is None
    ck = CheckpointManager(svc, str(tmp_path / "bk"), keep=5)
    assert ck.save() == 1
    svc.apply_updates({"edges": {"click": {"src": [30], "dst": [1], "ts": [99]}}})        # grows the table past the snapshot
    assert ck.save() == 2
    assert svc.delete_vertices("u", [1]) == 3 + 0 and st.get(1)[0].numel() == 0 and svc.vstores["u"].get_vertex(1) is None
    assert svc.run_query(0, [1])["hops"][0]["ids"].tolist() == [[-1, -1, -1]]
    assert svc.delete_edges("click", [2, 2, 777]) == 1
    assert [b["id"] for b in ck.list_backups()] == [1, 2] and all(b["bytes"] > 0 for b in ck.list_backups())
    assert ck.restore(1) == 1
    assert st.get(1)[0].tolist() == [4, 6, 5] and st.get(2)[0].tolist() == [7] and st.get(30)[0].numel() == 0
    assert ck.restore_latest() == 2 and st.get(30)[0].tolist() == [1]
    import pytest as _pt
    with _pt.raises(FileNotFoundError):
        ck.restore(9)
    assert ck.purge(keep=1) == 1 and [b["id"] for b in ck.list_backups()] == [2]


def test_native_record_parser_matches_python_loader(tmp_path):
    """csrc/host_loader.cpp parse_records (columnar batches straight from the file) vs the line-by-line Python loader: same
    service state for vertices with list + scalar attributes, weighted / unweighted and reversed edges, skipped lines, CRLF
    line ends, a missing final newline and batch sizes that cut the file into many windows."""
    from graphlearn_b200.dgs import FileLoader, Schema
    schema = Schema({
        "attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}, {"type": 1, "name": "weight", "value_type": "FLOAT32"},
                      {"type": 2, "name": "feature", "value_type": "FLOAT32_LIST"}, {"type": 3, "name": "age", "value_type": "FLOAT32"}],
        "vertex_defs": [{"vtype": 0, "name": "user", "attr_types": [0, 3, 2]}, {"vtype": 1, "name": "item", "attr_types": [0, 2]}],
        "edge_defs": [{"etype": 2, "name": "u2i", "attr_types": [0, 1]}, {"etype": 3, "name": "i2u", "attr_types": [0, 1]},
                      {"etype": 4, "name": "i2i", "attr_types": [0]}],
        "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}, {"etype": 3, "src_vtype": 1, "dst_vtype": 0},
                               {"etype": 4, "src_vtype": 1, "dst_vtype": 1}]})
    (tmp_path / "pattern").write_text("#VERTEX:user,vid,timestamp,feature,age\n#VERTEX:item,vid,feature,timestamp\n"
                                      "#EDGE:u2i,src,dst,timestamp,weight\n#EDGE:i2i,src,dst,timestamp\n# a comment\n")
    rs = np.random.RandomState(1)
    lines = []
    for i in range(700):
        r = rs.randint(0, 6)
        if r == 0:
            lines.append("user,%d,%d,%.3f:%.3f:%.3f,%d" % (rs.randint(0, 50), i, rs.rand(), rs.rand(), rs.rand(), rs.randint(18, 80)))
        elif r == 1:
            lines.append("item,%d,%.2f:%.2f,%d" % (rs.randint(0, 80), rs.rand(), rs.rand(), i))
        elif r in (2, 3):
            lines.append("u2i,%d,%d,%d,%.2f" % (rs.randint(0, 50), rs.randint(0, 80), rs.randint(0, 5000), rs.rand()))
        elif r == 4:
            lines.append("i2i,%d,%d,%d" % (rs.randint(0, 80), rs.randint(0, 80), rs.randint(0, 5000)))
        else:
            lines.append(["unknown,1,2,3", "u2i,1,2", "", "item,3,0.5:0.5,7,extra"][rs.randint(0, 4)])      # all skipped
    data = tmp_path / "data"
    data.write_bytes(("\r\n".join(lines[:350]) + "\r\n" + "\n".join(lines[350:])).encode())               # CRLF half, no final newline

    def build(native, bs):
        svc = DynamicGraphService(schema.to_service_schema(capacity=8, feat_dims={"user": 4, "item": 2}), device="cpu")
        svc.install_query(0, QueryPlan("user").out("u2i", 4).out("i2u", 3))
        svc.install_query(1, QueryPlan("item").out("i2i", 5))
        n = FileLoader(str(tmp_path / "pattern"), schema, batch_size=bs, reverse_edges={"u2i": "i2u"}, native=native).load(str(data), svc)
        return svc, n
    ref, n_ref = build(False, 64)
    want = {"user": 5, "item": 4, "u2i": 5, "i2i": 4}
    assert n_ref == sum(1 for l in lines if want.get(l.split(",")[0]) == len(l.split(",")))
    for bs in (64, 7, 100000):
        nat, n_nat = build(True, bs)
        assert n_nat == n_ref
        for et in ("u2i", "i2u", "i2i"):
            a, b = ref.stores[et], nat.stores[et]
            m = min(a.n, b.n)
            assert torch.equal(a.count[:m], b.count[:m]) and int(a.count[m:].sum()) == 0 and int(b.count[m:].sum()) == 0
            # same kept (timestamp, neighbour, weight) multisets per vertex; ties may sit in different slots
            for v in range(m):
                ka = sorted(zip(*(x.tolist() for x in a.get(v))))
                kb = sorted(zip(*(x.tolist() for x in b.get(v))))
                assert [x[1] for x in ka] == [x[1] for x in kb], (et, v)
        for vt in ("user", "item"):
            a, b = ref.vstores[vt], nat.vstores[vt]
            m = min(a.n, b.n)
            assert torch.equal(a.feat_ts[:m], b.feat_ts[:m])
            assert torch.allclose(a.feat[:m], b.feat[:m]) and float(a.feat[:m].abs().sum()) > 0       # vertex timestamps are unique
            if vt == "user":                                        # schema order (age, feature), not pattern order
                v = int((a.feat_ts > -(2 ** 61)).nonzero()[0])
                assert float(a.feat[v, 0]) >= 18
    # malformed numbers are errors, not silently dropped records
    (tmp_path / "bad").write_text("u2i,1,x,3,0.5\n")
    with pytest.raises(RuntimeError):
        FileLoader(str(tmp_path / "pattern"), schema, native=True).load(str(tmp_path / "bad"), ref)


def test_admin_token_and_service_side_load(tmp_path):
    """POST /admin/* needs the bearer token when the front end has one; /infer and read-only GETs stay open; the client sends
    the token; /admin/load bulk-loads a server-side record file; client.ingest / set_barrier round trip."""
    from graphlearn_b200.dgs import HttpFrontEnd, Schema
    from graphlearn_b200.dgs import client as C
    schema = Schema({"attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}],
                     "vertex_defs": [{"vtype": 0, "name": "u", "attr_types": [0]}, {"vtype": 1, "name": "i", "attr_types": [0]}],
                     "edge_defs": [{"etype": 2, "name": "e", "attr_types": [0]}],
                     "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}]})
    svc = DynamicGraphService(schema.to_service_schema(capacity=16), device="cpu")
    front = HttpFrontEnd(svc, schema, admin_token="s3cret").start()
    try:
        anon = C.Graph.connect("127.0.0.1:%d" % front.port)
        q = anon.V("u").feed(C.DataSource([1])).outV("e").sample(2).by("topk_by_timestamp").alias("h").values()
        st = anon.install(q)
        assert not st.ok() and "401" in st.message
        with pytest.raises(C.UserException):
            anon.ingest({"edges": {"e": {"src": [1], "dst": [2], "ts": [3]}}})
        assert anon.stats()["ingested"] == 0                             # open read-only surface
        g = C.Graph.connect("127.0.0.1:%d" % front.port, admin_token="s3cret")
        assert g.install(q).ok()
        (tmp_path / "pattern").write_text("#EDGE:e,src,dst,timestamp\n")
        (tmp_path / "data").write_text("e,1,5,10\ne,1,6,11\ne,1,7,12\n")
        assert g.load_file(str(tmp_path / "pattern"), str(tmp_path / "data")) == 3
        assert g.ingest({"edges": {"e": {"src": np.array([1]), "dst": np.array([9]), "ts": np.array([13])}}}) == 4
        g.set_barrier("b")
        assert g.check_barrier("b").ok()
        g.set_barrier("later", after_records=100)
        assert not anon.check_barrier("later").ok()
        assert anon.run(q)["h"]["ids"].tolist() == [[9, 7]]              # inference needs no token
    finally:
        front.stop()


def test_native_record_parser_fuzz_matches_python(tmp_path):
    """Randomised record files (signed / huge ids, '+' prefixes, exponent and bare-dot floats, empty list tokens, junk and
    short lines, CRLF or LF, with / without a final newline, batch sizes 1 / 3 / 1000): the native parser and the Python
    loader must produce identical batches - or fail alike."""
    import random
    from graphlearn_b200.dgs import FileLoader, Schema
    schema = Schema({
        "attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}, {"type": 1, "name": "weight", "value_type": "FLOAT32"},
                      {"type": 2, "name": "feature", "value_type": "FLOAT32_LIST"}, {"type": 3, "name": "age", "value_type": "FLOAT32"}],
        "vertex_defs": [{"vtype": 0, "name": "user", "attr_types": [0, 3, 2]}, {"vtype": 1, "name": "item", "attr_types": [0, 2]}],
        "edge_defs": [{"etype": 2, "name": "u2i", "attr_types": [0, 1]}, {"etype": 4, "name": "i2i", "attr_types": [0]}],
        "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}, {"etype": 4, "src_vtype": 1, "dst_vtype": 1}]})

    class Rec(object):
        def __init__(self):
            self.b = []

        def apply_updates(self, batch):
            self.b.append(batch)

    def flat(batches):
        out = {}
        for b in batches:
            for k, e in b["edges"].items():
                for s, d_, t, w in zip(e["src"], e["dst"], e["ts"], e["weight"]):
                    out.setdefault(("E", k), []).append((int(s), int(d_), int(t), round(float(w), 5)))
            for k, v in b["vertices"].items():
                for i, t, f in zip(v["id"], v["ts"], v["feat"]):
                    out.setdefault(("V", k), []).append((int(i), int(t), tuple(round(float(x), 4) for x in f)))
        return out
    d = str(tmp_path)
    with open(d + "/pattern", "w") as f:
        f.write("#VERTEX:user,vid,timestamp,feature,age\n#VERTEX:item,vid,feature,timestamp\n#EDGE:u2i,src,dst,timestamp,weight\n#EDGE:i2i,src,dst,timestamp\n")
    for seed in range(80):
        rs = random.Random(seed)
        num = lambda: rs.choice(["%d" % rs.randint(-5, 50), "+%d" % rs.randint(0, 9), "%d" % rs.randint(0, 10 ** 12)])  # noqa: E731
        fl = lambda: rs.choice(["%.3f" % rs.uniform(-2, 2), "1e-3", "+0.5", "%d" % rs.randint(0, 9), ".5", "5."])  # noqa: E731
        lines = []
        for _ in range(rs.randint(0, 60)):
            r = rs.randint(0, 7)
            if r == 0:
                lines.append("user,%s,%s,%s:%s:%s,%s" % (num(), num(), fl(), fl(), fl(), fl()))
            elif r == 1:
                lines.append("item,%s,%s:%s,%s" % (num(), fl(), fl(), num()))
            elif r in (2, 3):
                lines.append("u2i,%s,%s,%s,%s" % (num(), num(), num(), fl()))
            elif r == 4:
                lines.append("i2i,%s,%s,%s" % (num(), num(), num()))
            elif r == 5:
                lines.append(rs.choice(["", "junk", "u2i,1", "item,1,2,3,4,5", ",,,", "user", " "]))
            elif r == 6:
                lines.append("item,%s,%s::%s,%s" % (num(), fl(), fl(), num()))
            else:
                lines.append("u2i,%s,%s,%s,%s " % (num(), num(), num(), fl()))
        eol = rs.choice(["\n", "\r\n"])
        with open(d + "/data", "wb") as f:
            f.write((eol.join(lines) + (eol if rs.random() < 0.5 else "")).encode())
        res = []
        for native in (False, True):
            rec = Rec()
            try:
                n = FileLoader(d + "/pattern", schema, batch_size=rs.choice([1, 3, 1000]), native=native).load(d + "/data", rec)
                res.append((n, flat(rec.b)))
            except Exception as e:  # noqa: BLE001
                res.append(("ERR", type(e).__name__ in ("ValueError", "RuntimeError")))
        assert res[0] == res[1], (seed, lines)


def test_remote_data_loader_sdk():
    """dgs.client.data_loader (the reference's data-loader SDK: Initialize(dgs_host) + GroupProducer): records added on the client
    are batched, shipped to the service over HTTP, and become visible to queries once the barrier is READY."""
    from graphlearn_b200.dgs import HttpFrontEnd, Schema
    from graphlearn_b200.dgs import client as C
    schema = Schema({"attr_defs": [{"type": 0, "name": "timestamp", "value_type": "INT64"}, {"type": 1, "name": "f", "value_type": "FLOAT32_LIST"}],
                     "vertex_defs": [{"vtype": 0, "name": "u", "attr_types": [0, 1]}, {"vtype": 1, "name": "i", "attr_types": [0, 1]}],
                     "edge_defs": [{"etype": 2, "name": "e", "attr_types": [0]}],
                     "edge_relation_defs": [{"etype": 2, "src_vtype": 0, "dst_vtype": 1}]})
    svc = DynamicGraphService(schema.to_service_schema(capacity=16, feat_dims={"u": 2, "i": 2}), device="cpu")
    front = HttpFrontEnd(svc, schema).start()
    try:
        producer, g = C.data_loader("127.0.0.1:%d" % front.port, max_batch_size=5)
        q = g.V("u").feed(C.DataSource([2])).properties(1).alias("s").outV("e").sample(3).by("topk_by_timestamp").properties(1).alias("h").values()
        assert g.install(q).ok()
        producer.add_vertex("u", 2, 1, [0.5, 1.5])
        for i in range(7):
            producer.add_vertex("i", i, 1, [float(i), 0.0])
            producer.add_edge("e", 2, i, 100 + i)
        assert 0 < svc.ingested < 15 and producer.produced >= 10            # full batches already left the client
        producer.set_barrier(producer.sink, "all")
        assert g.check_barrier("all").ok() and svc.ingested == 7            # edges counted by the service (vertices are upserts)
        v = g.run(q)
        assert v["h"]["ids"].tolist() == [[6, 5, 4]] and v["h"]["features"][0, 0].tolist() == [6.0, 0.0]
        assert v["s"]["features"].tolist() == [[0.5, 1.5]]
    finally:
        front.stop()


def test_reference_dgs_conf_files_load():
    """The reference's own service configuration files (dynamic_graph_service/conf/{u2i,dblp,ut}: schema JSON, install-query JSON incl.
    the parameter-less SOURCE node of conf/dblp, YAML option files) drive this service unchanged.  Skipped without a checkout."""
    import glob
    import json
    import os
    from graphlearn_b200.dgs import Options, Schema
    base = os.path.join(os.environ.get("GLB_REFERENCE_DIR", ""), "dynamic_graph_service", "conf")
    if not os.path.isdir(base):
        pytest.skip("no reference checkout")
    want = {"u2i": [("u2i", 10), ("i2i", 5)], "dblp": [("published", 5), ("written", 5)]}
    for name in ("u2i", "dblp", "ut"):
        sch = Schema.from_json(os.path.join(base, name, "schema.%s.json" % name))
        iq = json.load(open(os.path.join(base, name, "install_query.%s.json" % name)))
        plan = QueryPlan.from_json(iq, sch)
        svc = DynamicGraphService(sch.to_service_schema(capacity=8), device="cpu")
        svc.install_query(int(iq.get("query_id", 0)), plan)
        if name in want:
            assert plan.hops == want[name]
        src_type = plan.source_type
        first = plan.edge_nodes()[0].etype
        svc.apply_updates({"edges": {first: {"src": [1, 1], "dst": [2, 3], "ts": [5, 6]}}})
        assert svc.run_query(int(iq.get("query_id", 0)), [1])["hops"][0]["ids"][0, 0].item() == 3 and src_type in sch.vertex_id
    for y in glob.glob(os.path.join(base, "ut", "*.yml")):
        assert Options.from_yaml(y).get("http-port") is not None
