"""Hand-scheduled training step for EgoGraphSAGE (any depth; mean, sum, max or gcn aggregation).

Same math as ``models.graphsage.EgoGraphSAGE`` + ``SageTrainer``'s autograd
path, but forward and backward are an explicit, minimal kernel chain over
pre-allocated buffers (static shapes -> CUDA graph friendly):

  K1    sample hop 1..L of the NEXT batch (parallel branch)            (L launches + 1 counter kernel)
  K6+K7 ONE persistent launch per layer: gather / aggregate / wgmma GEMM of every hop pair of the layer
        (multi-segment); the top layer's launch also computes softmax-CE, dlogits and the bias gradient
  for l = L..1:  dW_l = dZ_l^T A_l   split-K wgmma kernel, fp32 accumulation straight into the flat gradient buffer;
                                     for l < L, dZ_l = relu'(H_l) * (self + nbr/k rows of dA_{l+1}) is computed by its producers
                                     (gcn above: both parts scaled by 1/(k+1); max above: the neighbour part of a column
                                     reaches only the child that held its max, from the argmax bytes of layer l+1's forward)
                 dA_l = dZ_l W_l     [l > 1] mma.sync kernel over the layer's forward weight images
  K8    ONE kernel: peer-memory all-reduce (world > 1) + Adam + gradient zeroing + bf16 weight images of the next step
        (+ the dropout step counter when p > 0)

Dropout (``model.dropout = p``, read once at construction; it is part of the captured graphs): the output of every
hidden layer l < L is ``H_l = relu(Z_l) * m / (1 - p)`` with m ~ Bernoulli(1 - p) per element, as the reference's EgoGNN
drops each hidden hop tensor once after the activation.  A row of H_l is both a self row and a neighbour row of layer
l + 1, and both read the same dropped value.  Neither the layer-1 input features nor the top layer (logits,
embeddings) are dropped, and ``infer_all`` / ``evaluate`` / ``predict`` / ``embed`` never drop.  The mask is drawn in
the forward epilogue (after bias and ReLU, before the bf16 store) and is a pure function of (dropout seed, step
counter, layer l, row of the layer's output buffer, output column) - see ``dropout_bits`` in csrc/sage_fused.cu.  The
seed is the sampler's per-rank seed with its own salt; the counter is advanced by ``adam_pack`` after every forward
launch of the step.  No mask is stored: H_l > 0 exactly where m * relu'(Z_l) = 1, so the dW kernel's relu'(H_l) test
applies the mask and ``sage_bwd_da`` of layer l + 1 applies the 1 / (1 - p).

Learned input embedding (``learn_input_embedding=True``): layer 1 reads a trainable table E ``[n_local, d]`` through a
bf16 image, as it reads a feature table otherwise.  Without float attributes, d is the first layer's input width.  With
f = ``nodes.float_dim`` > 0 float attributes, layer 1's input row is ``[E_r || x_r]``, d = in_dim - f: image columns
[0, d) hold E and [d, d + f) the attributes rounded to bf16, and the columns of each half of W_1 follow that order.  The
attribute columns are a snapshot taken at construction (training never writes them; a later ``set_float`` on the node
table is not seen).  The backward adds three launches: dW_1 also stores dZ_1 (and a max layer 1's forward its argmax
bytes), dA_1 = dZ_1 W_1 runs on ``sage_bwd_da`` (with attributes: only over the 64-column blocks that hold E's columns),
and ``embed_grad_scatter`` adds the self / neighbour halves of dA_1 (scaled like the layer's aggregator) into an fp32
gradient table and marks the rows read in a bitmap.  ``embed_lazy_adam`` then updates the touched rows only
(``torch.optim.SparseAdam``'s semantics at the dense Adam's step count), rewrites their E columns of the image and
clears their gradient rows and bits, on a branch beside ``adam_pack``.

Batch normalisation (``EgoGraphSAGE(batch_norm=True)``, one ``BatchNorm1d`` per hidden layer in ``model.norms``): every
hop tensor (segment) of hidden layer l is ``H_l = dropout(relu(BN_l(Z_l)))``, normalised with its own batch mean and
biased variance, and the running statistics are updated once per segment in hop order, as the reference's EgoGNN
calls bn_func once per hop tensor.  The hidden layer's launch writes Z_l in fp32 (its conv has no bias, no ReLU, no
dropout), and csrc/sage_bn.cu adds per BN layer:
  forward   bn_colsum<false>  per-segment mean / rstd (shifted sums) + the module's running buffers, in place
            bn_apply          H_l = dropout(relu(gamma x^ + beta)) in bf16, the epilogue's dropout mask
  backward  sage_bwd_dz       sage_bwd_dw's dZ-only mode: dY_l, the routed gradient of the BN output, in bf16
            bn_colsum<true>   per-segment sum(dY), sum(dY x^); d gamma, d beta into the flat gradient buffer
            bn_bwd_apply      dZ_l in bf16, then dW_l on the dense dZ path (beside dA_l) and dA_l as without BN
``infer_all`` / ``evaluate`` fold the eval-mode BN into inference-only weight images and bias; ``predict`` / ``embed``
run the model's eval-mode autograd path.  Both use the running statistics.

Wide layers (``ops.sage.fused_layer_plan``): a mean, sum or max layer whose padded K = 2 kp (inputs 257-512 wide: K =
1024) does not fit one CTA's shared memory runs split-K, as two launches of the same persistent kernel: the self half
(no neighbours) writes x_self . W_self^T into an fp32 partial P and A[:, :kp], the neighbour half gathers and aggregates,
fills A[:, kp:], adds P to its accumulators and runs the layer's epilogue (bias, ReLU, dropout, argmax bytes) exactly as
one launch would.  The images are the layer's usual ones (each half is a k-block range of every image), so the backward
and the fused Adam kernel see an ordinary layer with K = 2 kp.  A split top layer computes its loss with ``softmax_ce``.

9 launches of this repo's kernels (0 library kernels) for the 2-layer flagship instead of ~60 on the autograd path
(12 with the learned input embedding, 14 with batch normalisation; one more per split-K layer, and one more when the
top layer is split, for its loss kernel).
Layer l consumes hop pairs (i, i+1) for i in 0..L-l, exactly the EgoGNN
recursion of graphlearn/python/nn/tf/model/ego_gnn.py:58-110.

Scheduling (see ``_step_body`` / ``capture``): the launches above form a DAG, not a chain - independent ones
run on forked streams, which become parallel branches of the captured CUDA graph; under capture the step is
additionally software pipelined: graph replay t trains on the batch that replay t-1 staged (pinned host ->
device) and sampled on a side branch, and the loss leaves through another branch.  Public API: ``capture()``,
``step(seed_ids_host)`` (end to end), ``step_device()`` (no host traffic), ``from_query`` / ``step_query`` (driven by a
compiled GSL query), ``predict``, ``state_dict``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch

from ..ops import comm as comm_ops
from ..ops import rng as rng_ops
from ..ops import sage as sage_ops
from ..ops import sampling as S
from ..parallel.runtime import Runtime, local_table_desc, native
from ..store.shards import CsrShard, NodeTable


@dataclass
class HiddenBatchNorm:
    """Batch normalisation of a hidden layer (``EgoGraphSAGE(batch_norm=True)``): the layer's launch writes Z (fp32, no
    bias, no ReLU) and ``H = dropout(relu(BN(Z)))`` follows per segment with the segment's own batch statistics."""
    norm: torch.nn.BatchNorm1d      # the model's module: gamma / beta (views of flat_p / flat_g) and the running buffers,
                                    # which the forward statistics kernel updates in place
    Z: torch.Tensor                 # fp32 [rows, out_dim], columns laid out as Hp's (N-split: image i at i * N)
    mean: torch.Tensor              # fp32 [nseg, out_dim] batch mean of each segment
    rstd: torch.Tensor              # fp32 [nseg, out_dim] 1 / sqrt(biased variance + eps)
    gsum: torch.Tensor              # fp32 [nseg, 2, out_dim] backward: sum(dY), sum(dY x^) per segment
    dY: torch.Tensor                # bf16 [rows, out_dim] gradient of the BN output (ReLU, dropout and routing applied)
    tickets: torch.Tensor           # int32 [2, ceil(out_dim / 64)] zero between launches (forward / backward column sums)
    drop: tuple                     # bn_fwd_apply's (drop_state, drop_p, drop_layer): dropout of H (p > 0), else off


@dataclass
class SageLayer:
    """Layer l (1-based) of a ``FastSageTrainer``, described once at construction: shape facts, buffers and the launch
    arguments that do not change between steps.  The layer runs the hop pairs (i, i + 1), i = 0..nseg - 1, as the
    segments of one launch; segment i is the rows ``offs[i]:offs[i + 1]`` of each of its buffers."""
    conv: torch.nn.Module
    last: bool
    mode: int                       # sage_ops.MODE of the aggregation
    kt: int                         # padded K: columns of weight_p and of the A / dA rows
    ns: int                         # forward weight images (N-split when W does not fit next to the A tiles)
    N: int                          # padded output columns per image
    n_out: int                      # columns one image writes: out_dim, or N when the layer is N-split
    nseg: int
    offs: List[int]
    rows: int
    fuse_ce: bool                   # the forward launch computes softmax-CE, dZ and the bias gradient in its epilogue
    Hp: torch.Tensor                # output with the rows padded to the image columns (bf16; top layer fp32 logits)
    H: torch.Tensor                 # ... its out_dim real columns
    A: torch.Tensor                 # saved [self || agg] tiles (bf16)
    dZp: torch.Tensor               # dZ with the row padded to the K padding of the dA GEMM
    dZ: torch.Tensor
    dA: Optional[torch.Tensor]      # None for layer 1, unless it reads the learned input table
    img: torch.Tensor               # bf16 weight images (rewritten by the fused Adam kernel at the end of every step)
    dW: torch.Tensor                # the weight's and the bias's views of the flat gradient buffer
    db: Optional[torch.Tensor]
    below: Optional[torch.Tensor]   # table descriptor of H of the layer below; None for layer 1 (feature table, hop ids)
    fwd: tuple                      # sage_fused_multi's (self_base, nbr_base, Ms, ks, outs, a_saves)
    # sage_fused_multi's (drop_state, drop_p, drop_layer, drop_row0): dropout of this layer's output (hidden layers with
    # p > 0; (None, 0.0, 0, []) otherwise)
    drop: tuple
    da_alpha: float                 # scale of dA: 1 / (1 - p) when the layer's input H_{l-1} is dropped out, else 1
    # sage_bwd_da's kb_ranges: the 64-column blocks of dA it computes, () = all (layer 1 with a learned input embedding
    # next to float attributes: only E's blocks of each half, nobody reads the attributes' gradient)
    da_blocks: tuple = ()
    # max aggregation, l >= 2: uint8 [rows, in_nbr padded to 16], row m of segment i = for each neighbour-half column the
    # first of the k neighbours holding its max, written by the forward (`amax` per-segment views) for the layer below's
    # gradient routing; layer 1 has them only when it reads the learned input table (a feature table has no gradient)
    argmax: Optional[torch.Tensor] = None
    amax: list = None
    # split-K forward (a mean / sum / max layer whose padded K = kt does not fit one launch): the self half writes
    # x_self . W_self^T into P (fp32, columns as Hp's) and A[:, :kt / 2]; the neighbour half (`fwd`, `drop`, `amax`) fills
    # A[:, kt / 2:], adds P and runs the epilogue.  fwd_self = the self half's (self_base, nbr_base, Ms, ks, outs, a_saves)
    split: bool = False
    P: Optional[torch.Tensor] = None
    fwd_self: Optional[tuple] = None
    # sage_bwd_dw's keyword arguments (seg_row0, seg_row1, self_src, nbr_src, seg_k, seg_scale, nbr_col0, dz_out,
    # seg_self_scale, amax_src) for l < L, where dZ_l is computed from dA of the layer above (with batch norm: dY, the
    # gradient of the BN output, into bn.dY)
    bwd: Optional[dict] = None
    bn: Optional[HiddenBatchNorm] = None


@dataclass
class InputEmbedding:
    """The learned layer-1 input table E ``[n_local, d]`` of a trainer built with ``learn_input_embedding=True``: row r
    is the node with vid ``r * world + rank``.  Layer 1 reads the bf16 image ``[E || x]`` (x: the node table's f float
    attributes, f = 0 without them); the fp32 tables (master, Adam moments, gradient) have ``dp = d`` rounded up to 8
    columns, whose padding stays zero (with attributes d is a multiple of 8, so dp = d)."""
    d: int
    f: int
    table: object                   # SymmTensor: bf16 image [n_local, stride] (E in [0, d), x in [d, d + f)), stride by
                                    # the feature tables' rules
    desc: torch.Tensor              # its table descriptor (what layer 1 reads where a feature table's is read otherwise)
    view: object                    # NodeTable-like (rt, feats, feat_desc, float_dim) over the image: predict / embed
    master: torch.Tensor            # fp32 [n_local, dp]
    m: torch.Tensor
    v: torch.Tensor
    grad: torch.Tensor              # fp32 [n_local, dp], scattered by embed_grad_scatter, zeroed row by row by the update
    bits: torch.Tensor              # int32 [ceil(n_local / 32)]: rows touched by the step (cleared by the update)
    lr: float
    scatter: dict                   # embed_grad_scatter's per-layout arguments (seg_row0, seg_k, self_scale, nbr_scale, ...)


class FastSageTrainer:
    def __init__(self, rt: Runtime, nodes: NodeTable, csr: CsrShard, model, fanouts: Sequence[int], batch_size: int,
                 lr: float = 3e-3, strategy: str = "random", use_cuda_graph: bool = True, allreduce: str = "peer",
                 seed: int = 0, allreduce_dtype: str = "fp32", learn_input_embedding: bool = False,
                 embedding_lr: Optional[float] = None):
        self.ar_bf16 = allreduce_dtype == "bf16"      # stage the gradient exchange in bf16 (halves the NVLink bytes)
        assert rt.is_cuda, "FastSageTrainer is the CUDA engine; use SageTrainer for the portable path"
        self.rt, self.nodes, self.csr, self.model = rt, nodes, csr, model
        self.fanouts = list(fanouts)
        self.L = len(self.fanouts)
        assert self.L == model.num_layers
        self.B = int(batch_size)
        self.dropout = float(getattr(model, "dropout", 0.0))
        if not 0.0 <= self.dropout < 1.0:
            raise ValueError("dropout must be in [0, 1), got %r" % (self.dropout,))
        if learn_input_embedding:
            self._check_input_embedding(rt, nodes, model, self.fanouts)
        self.batch_norm = bool(getattr(model, "batch_norm", False))
        if self.batch_norm and rt.world > 1:
            raise ValueError("batch_norm trains on one GPU only (world = %d)" % rt.world)
        if self.batch_norm and self.B < 2:
            raise ValueError("batch_norm needs at least 2 rows per hop tensor (batch of %d roots)" % self.B)
        self.strategy = strategy
        self.C = native()
        dev = rt.device
        self.rng = rng_ops.DeviceRng(rt, seed)
        # dropout masks: {seed, step counter}; the seed is the sampler's per-rank seed with its own salt, the counter is
        # advanced by adam_pack once per step (never by the sampling branch, which runs beside the forward under capture)
        self.drop_state = torch.tensor([(self.rng.seed * 0x9E3779B1 + self.DROPOUT_SALT) % 2 ** 63, 0],
                                       dtype=torch.int64, device=dev)
        self._drop_ctr = self.drop_state[1:] if self.dropout > 0 else None
        self.flat_p, self.flat_g = comm_ops.flatten_module(model)
        if rt.world > 1:            # replicas start from rank 0's initialisation (what DDP does at construction)
            import torch.distributed as dist
            with torch.no_grad():
                dist.broadcast(self.flat_p, src=0)
        self.opt = comm_ops.FlatAdam(self.flat_p, self.flat_g, lr=lr)
        self.ar = comm_ops.PeerAllReduce(rt, self.flat_g.numel(), backend=allreduce)
        self.seeds = torch.zeros(self.B, dtype=torch.int64, device=dev)
        self.g_store = model._glb_grad_storage            # grads + 4 scratch floats, zeroed by ONE memset
        self.loss = self.g_store[self.flat_g.numel():self.flat_g.numel() + 1]
        # hop sizes n_i = B * prod(k_j, j < i)
        self.n = [self.B]
        for k in self.fanouts:
            self.n.append(self.n[-1] * k)
        self.convs = list(model.convs)
        self.layers: List[SageLayer] = []
        for l, c in enumerate(self.convs, 1):
            assert c.agg_type in ("mean", "sum", "max", "gcn"), "fast engine supports mean / sum / max / gcn aggregation"
            last = l == self.L
            kt = c.weight_p.size(1)
            halves, ns, N = sage_ops.fused_layer_plan(c.in_self, c.in_nbr, c.out_dim, c.agg_type, max(self.fanouts),
                                                      last=last)
            n_out = c.out_dim if ns == 1 else N
            nseg = self.L - l + 1
            offs = [0]
            for i in range(nseg):
                offs.append(offs[-1] + self.n[i])
            rows = offs[-1]
            Hp = torch.zeros(rows, ns * N if last else c.out_dim, dtype=torch.float32 if last else torch.bfloat16, device=dev)
            A = torch.zeros(rows, kt, dtype=torch.bfloat16, device=dev)
            dZp = torch.zeros(rows, sage_ops.pad_k(c.out_dim), dtype=torch.bfloat16, device=dev)
            # (layer 1 has a dA, and a max layer 1 its argmax bytes, only when its input is the learned table)
            dA = torch.zeros(rows, kt, dtype=torch.bfloat16, device=dev) if l > 1 or learn_input_embedding else None
            argmax = None
            if (l > 1 or learn_input_embedding) and c.agg_type == "max":
                argmax = torch.zeros(rows, (c.in_nbr + 15) // 16 * 16, dtype=torch.uint8, device=dev)
            below, self_base, nbr_base = None, [0] * nseg, [0] * nseg
            if l > 1:
                # the segments' self / neighbour rows are the contiguous row ranges of segments i / i + 1 of the layer
                # below, which in turn takes dZ of its segment s from the self rows of segment s and the neighbour
                # rows of segment s - 1 of this layer's dA
                lo = self.layers[-1]
                below, self_base, nbr_base = local_table_desc(lo.H), lo.offs[:nseg], lo.offs[1:nseg + 1]
                da_seg = [dA[offs[i]:offs[i + 1]] for i in range(nseg)]
                k_nbr = self.fanouts[:nseg]
                gcn = c.agg_type == "gcn"
                scale = [1.0 / k if c.agg_type == "mean" else 1.0 / (k + 1) if gcn else 1.0 for k in k_nbr]
                # gcn: the self row is one of the k + 1 rows of the mean; max: the argmax rows of the parents
                self_scale = [1.0 / (k + 1) for k in k_nbr] + [1.0] if gcn else []
                amax_src = [None] + [argmax[offs[i]:offs[i + 1]] for i in range(nseg)] if argmax is not None else []
                lo.bwd = dict(seg_row0=lo.offs[:-1], seg_row1=lo.offs[1:], self_src=da_seg + [None], nbr_src=[None] + da_seg,
                              seg_k=[1] + k_nbr, seg_scale=[1.0] + scale,
                              nbr_col0=sage_ops.padded_dims(c.in_self, c.in_nbr, c.agg_type)[0],
                              dz_out=lo.bn.dY if lo.bn is not None else lo.dZ if lo.dA is not None else None,
                              seg_self_scale=self_scale, amax_src=amax_src)
            bn = None
            if self.batch_norm and not last:
                # the launch writes Z; dropout moves to the BN apply kernel, which draws the epilogue's mask
                Z = torch.zeros(rows, c.out_dim, dtype=torch.float32, device=dev)
                bn = HiddenBatchNorm(
                    norm=model.norms[l - 1], Z=Z,
                    mean=torch.zeros(nseg, c.out_dim, dtype=torch.float32, device=dev), rstd=torch.zeros(nseg, c.out_dim, device=dev),
                    gsum=torch.zeros(nseg, 2, c.out_dim, device=dev),
                    dY=torch.zeros(rows, c.out_dim, dtype=torch.bfloat16, device=dev),
                    tickets=torch.zeros(2, (c.out_dim + 63) // 64, dtype=torch.int32, device=dev),
                    drop=(self.drop_state, self.dropout, l) if self.dropout > 0 else (None, 0.0, 0))
            drop = (self.drop_state, self.dropout, l, offs[:-1]) if self.dropout > 0 and not last and bn is None \
                else (None, 0.0, 0, [])
            outs = [(Hp if bn is None else bn.Z)[offs[i]:offs[i + 1], :n_out] for i in range(nseg)]
            a_saves = [A[offs[i]:offs[i + 1]] for i in range(nseg)]
            split, P, fwd_self = halves == 2, None, None
            if split:
                kp = kt // 2
                P = torch.zeros(rows, ns * N, dtype=torch.float32, device=dev)
                fwd_self = (self_base, nbr_base, self.n[:nseg], [0] * nseg, [P[offs[i]:offs[i + 1], :n_out] for i in range(nseg)],
                            [a[:, :kp] for a in a_saves])
                a_saves = [a[:, kp:] for a in a_saves]
            self.layers.append(SageLayer(
                conv=c, last=last, mode=sage_ops.MODE[c.agg_type], kt=kt, ns=ns, N=N, n_out=n_out,
                nseg=nseg, offs=offs, rows=rows,
                fuse_ce=last and self._fuse_ce and ns == 1 and N <= 64 and not split,
                Hp=Hp, H=Hp[:, :c.out_dim], A=A, dZp=dZp, dZ=dZp[:, :c.out_dim], dA=dA,
                img=torch.zeros(kt * ns * N, dtype=torch.bfloat16, device=dev),
                dW=c.weight_p.grad, db=c.bias.grad if c.bias is not None else None,
                below=below, fwd=(self_base, nbr_base, self.n[:nseg], self.fanouts[:nseg], outs, a_saves),
                drop=drop, da_alpha=1.0 / (1.0 - self.dropout) if l > 1 else 1.0,
                argmax=argmax, amax=[] if argmax is None else [argmax[offs[i]:offs[i + 1]] for i in range(nseg)], bn=bn,
                split=split, P=P, fwd_self=fwd_self))
        self.emb: Optional[InputEmbedding] = None
        if learn_input_embedding:
            self.emb = self._make_input_embedding(lr if embedding_lr is None else float(embedding_lr))
        # the lists other code reads; they alias the records' tensors
        self.H = [ly.H for ly in self.layers]
        self.dA = [ly.dA for ly in self.layers]
        self.img = [ly.img for ly in self.layers]
        self.n_split = [ly.ns for ly in self.layers]
        self.n_img = [ly.N for ly in self.layers]
        # one row per weight for the fused Adam kernel, which rewrites the images at the end of every step
        self._mats = torch.tensor([[model._glb_param_offsets[id(ly.conv.weight_p)], ly.conv.out_dim, ly.kt, ly.N,
                                    ly.img.data_ptr()] for ly in self.layers], dtype=torch.int64)
        self.loss_out = torch.zeros(1, dtype=torch.float32, device=dev)
        self.repack()
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self._skip_opt = False          # tests: stop before the optimiser to inspect the gradients
        # training branches run at high priority: pending CTAs of the whole-SM persistent kernels must win SM slots
        # against the (low-priority) next-batch sampling branch
        self._side = torch.cuda.Stream(priority=-1)
        self._loss_stream = torch.cuda.Stream()          # end-to-end graphs: the loss -> pinned host copy
        self.use_graph = bool(use_cuda_graph)
        self._steps = 0
        # double-buffered pinned staging of step(): batch in, loss out
        self._h_seeds2 = [torch.zeros(self.B, dtype=torch.int64).pin_memory() for _ in range(2)]
        self._h_loss2 = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.h_loss = self._h_loss2[0]                  # the loss slot of the latest step()
        # device-side aliases of the pinned host buffers (cudaHostAlloc memory is UVA-mapped)
        self._h_seeds_dev = [self.C.tensor_from_ptr(t.data_ptr(), [self.B], 2, dev.index) for t in self._h_seeds2]
        self._h_loss_dev = [self.C.tensor_from_ptr(t.data_ptr(), [1], 0, dev.index) for t in self._h_loss2]
        self._e2e_done = [torch.cuda.Event() for _ in range(2)]
        for e in self._e2e_done:
            e.record()
        # root traversal driving step_query (installed by from_query / a subclass), its next-epoch prefetch thread
        self._q_iter = self._q_thread = self._q_next = None
        self._inf = None                # infer_all: (CSR plan, local vids, hidden-layer tables), built on first call

    # ------------------------------------------------------------------ learned input embedding
    EMBED_SALT = 0x454D4244         # salt of the input embedding's initialisation seed ("EMBD")

    @staticmethod
    def _check_input_embedding(rt: Runtime, nodes: NodeTable, model, fanouts: Sequence[int]):
        c = model.convs[0]
        f = nodes.float_dim
        if f > 0 and c.in_self <= f:
            raise ValueError("learn_input_embedding concatenates a learned embedding with the node table's %d float "
                             "attributes: the first layer's input width (%d) leaves no columns for it" % (f, c.in_self))
        if f > 0 and (c.in_self - f) % 8 != 0:
            raise ValueError("learn_input_embedding next to float attributes needs an embedding width (input width %d - "
                             "%d attributes = %d) that is a multiple of 8" % (c.in_self, f, c.in_self - f))
        if f > 0 and nodes.feats.local.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("learn_input_embedding reads float attributes from fp32 or bf16 node tables (this one stores "
                             "block-scaled fp8)")
        if c.in_self != c.in_nbr:
            raise ValueError("learn_input_embedding needs the first layer's self and neighbour input widths to be equal "
                             "(got %d and %d)" % (c.in_self, c.in_nbr))
        _, N = sage_ops.split_images(c.weight_p.size(1), c.out_dim)
        if c.in_self < 1 or not sage_ops.fused_supported(c.in_self, c.in_nbr, min(c.out_dim, N), c.agg_type, max(fanouts)):
            raise ValueError("learn_input_embedding: the fused layer does not run a %d-wide input with out_dim %d, %s "
                             "aggregation and fan-out %d" % (c.in_self, c.out_dim, c.agg_type, max(fanouts)))
        if rt.world > 1:
            raise ValueError("learn_input_embedding trains on one GPU only (world = %d)" % rt.world)

    def _make_input_embedding(self, lr: float) -> InputEmbedding:
        """E ~ truncated normal (+-2 sigma, sigma = 1 / sqrt(d)) from the trainer's seed with its own salt, the bf16
        image [E || x], Adam moments, gradient table and touched-row bitmap, and the scatter's arguments for layer 1's
        segments."""
        from .. import config as _config
        from ..ops.gather import gather_rows
        from ..parallel.runtime import make_table_desc
        from types import SimpleNamespace
        rt, nodes, dev = self.rt, self.nodes, self.rt.device
        n, f = nodes.n_local, nodes.float_dim
        ly = self.layers[0]
        c = ly.conv
        width = c.in_self                                           # d + f columns of a layer-1 input row
        d = width - f
        dp = (d + 7) // 8 * 8
        g = torch.Generator(device=dev).manual_seed((self.rng.seed * 0x9E3779B1 + self.EMBED_SALT) % 2 ** 63)
        sigma = d ** -0.5
        master = torch.zeros(n, dp, dtype=torch.float32, device=dev)
        torch.nn.init.trunc_normal_(master[:, :d], std=sigma, a=-2 * sigma, b=2 * sigma, generator=g)
        stride = (width + 7) // 8 * 8                               # 16-byte bf16 rows, line-aligned when wide (set_float)
        align = int(getattr(_config.get(), "feature_row_align", 128))
        if align > 16 and width * 2 > align // 2:
            stride = (width * 2 + align - 1) // align * align // 2
        table = rt.symm_empty((n, stride), torch.bfloat16)
        table.local.zero_()
        table.local[:, :dp] = master.to(torch.bfloat16)
        if f > 0:                   # the attributes, rounded to bf16 once (training never writes these columns)
            table.local[:, d:width] = gather_rows(rt, nodes.feats, nodes.feat_desc, nodes.idmap.local_vids(),
                                                  f).to(torch.bfloat16)
        desc = make_table_desc(rt.world, width, stride, torch.bfloat16, table.nrows, table.ptrs)
        k = self.fanouts[:ly.nseg]
        agg = c.agg_type
        sscale = [1.0 / (x + 1) if agg == "gcn" else 1.0 for x in k]
        nscale = [1.0 / x if agg == "mean" else 1.0 / (x + 1) if agg == "gcn" else 1.0 for x in k]
        nbr_col0 = sage_ops.padded_dims(width, width, agg)[0]
        scatter = dict(seg_row0=ly.offs[:-1], seg_k=k, self_scale=sscale, nbr_scale=nscale, nbr_col0=nbr_col0,
                       amax=ly.amax)
        if f > 0:
            # dA_1 over E's 64-column blocks of the self half [0, d) and of the neighbour half [nbr_col0, nbr_col0 + d)
            # (gcn: one shared half at column 0): the attributes' columns of dA_1 would be most of its bytes, unread
            nb = (d + 63) // 64
            ly.da_blocks = ((0, nb),) + (((nbr_col0 // 64, nbr_col0 // 64 + nb),) if nbr_col0 else ())
        return InputEmbedding(d=d, f=f, table=table, desc=desc,
                              view=SimpleNamespace(rt=rt, feats=table, feat_desc=desc, float_dim=width),
                              master=master, m=torch.zeros_like(master), v=torch.zeros_like(master),
                              grad=torch.zeros_like(master), bits=torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev),
                              lr=lr, scatter=scatter)

    def input_embedding(self) -> torch.Tensor:
        """The fp32 master copy of the learned input table E, ``[n_local, d]``, row r = the node with vid
        ``r * world + rank`` (``utils.checkpoint.save_embeddings`` exports it)."""
        if self.emb is None:
            raise ValueError("this trainer was built without learn_input_embedding")
        return self.emb.master[:, :self.emb.d]

    def _input_desc(self) -> torch.Tensor:
        """descriptor of the table layer 1 reads: the learned input table, or the node table's float attributes"""
        return self.nodes.feat_desc if self.emb is None else self.emb.desc

    # ------------------------------------------------------------------ GSL front end
    @classmethod
    def from_query(cls, graph, query, model, lr: float = 3e-3, **kw) -> "FastSageTrainer":
        """Train from a ``gl.Graph`` + GSL query (the API the reference trains through,
        graphlearn/python/gsl/dag_node.py:164-305, gsl/dag_dataset.py:29-97):

            q = g.V("i").batch(1024).shuffle(traverse=True).alias("src") \
                 .outV("e").sample(25).by("random").alias("h1").outV("e").sample(10).by("random").alias("h2").values()
            tr = FastSageTrainer.from_query(g, q, model); tr.capture()
            while True:
                try: loss = tr.step_query()
                except gl.OutOfRangeError: break        # end of epoch

        The query is compiled to a static sampling plan (gsl/compile.py); its hop chain becomes the sampling branch of
        the captured training-step graph, its root traversal (batch / shuffle / epochs) drives ``step_query``."""
        from ..gsl.compile import compilable, compile_query
        plan = compile_query(query)
        if plan is None or not compilable(graph, plan):
            raise ValueError("query cannot be lowered to a static sampling plan (need V().batch()[.shuffle()] followed by "
                             "outV/inV(...).sample(k).by(strategy) hops over dense-id node types on CUDA)")
        ets = {(h.edge_type, h.direction, h.strategy) for h in plan.hops}
        if len(ets) != 1:
            raise ValueError("the fused engine trains homogeneous chains: every hop must use the same edge type and strategy")
        et, direction, strategy = next(iter(ets))
        store = graph.store
        csr = store.reverse_csr(et) if direction == "in" else store.edges[et]
        if strategy == "in_degree" and direction == "out":
            store.ensure_indegree_weights(et)
        nodes = store.nodes[plan.base_type]
        if any(h.dst_type != plan.base_type for h in plan.hops):
            raise ValueError("the fused engine needs src and dst of the sampled edge type to be the root's node type")
        tr = cls(graph.runtime, nodes, csr, model, plan.fanouts, plan.batch_size, lr=lr, strategy=strategy, **kw)
        tr.plan, tr.graph_api = plan, graph
        rt = graph.runtime
        tab = store.nodes[plan.root_type]
        rows = tab.present.nonzero().flatten() if tab.present is not None else torch.arange(tab.n_local, device=rt.device)
        vids = rows * rt.world + rt.rank
        if plan.base_type != plan.root_type:
            vids = nodes.idmap.to_vid(tab.idmap.to_id(vids))
        tr._set_traversal(vids.cpu(), plan.batch_size, plan.traverse)
        return tr

    def _set_traversal(self, items: torch.Tensor, batch_size: int, strategy: str):
        """Make ``step_query`` walk the host tensor `items` (roots, or whatever the subclass's ``_fill_slot`` takes)
        in batches of `batch_size` with the GSL traversal `strategy`."""
        from .. import config as _config
        from ..gsl.iterators import SeedIterator
        self._q_vids = items
        # full batches only: the step graph has static shapes and the loss is normalised by B (the reference's PyTorch
        # loader also truncates every rank to min(count) // batch_size batches, examples/pytorch/gcn/train.py:174)
        self._q_iter = SeedIterator(int(items.numel()), batch_size, strategy, "cpu",
                                    seed=_config.get().seed + 17 * self.rt.rank, drop_last=True)
        self._q_refresh()

    def _q_refresh(self):
        """Per-epoch seed order: the root traversal's permutation applied to this rank's vids once per epoch, so that a
        step only slices it (host work per step stays at a few microseconds)."""
        it = self._q_iter
        if self._q_thread is not None:
            self._q_thread.join()
            self._q_thread = None
        nxt, self._q_next = self._q_next, None
        if it.strategy == "shuffle" and nxt is not None and nxt[0] == it.epoch and it._perm is None:
            it._perm, self._q_order = nxt[1], nxt[2]      # permutation of this epoch, prepared by the background thread
        elif it.strategy == "shuffle":
            self._q_order = self._q_vids[it.prime()]
        elif it.strategy == "by_order":
            self._q_order = self._q_vids
        else:
            self._q_order = None
        self._q_epoch = it.epoch

    def step_query(self) -> torch.Tensor:
        """One training step on the next seed batch of the compiled GSL query (host traversal -> pinned staging ->
        the step graph).  Raises ``OutOfRangeError`` at the end of an epoch, exactly like ``Dataset.next()``."""
        it = self._q_iter
        if self._q_epoch != it.epoch:
            self._q_refresh()
        if self._q_order is None:                       # 'random' traversal: draws with replacement
            return self._step_staged(self._q_vids[it.next_index()])
        lo = it.cursor
        it.next_index()                                  # advances the cursor / raises OutOfRangeError at the epoch end
        if it.strategy == "shuffle" and lo * 2 > it.n and self._q_thread is None and self._q_next is None:
            self._q_prefetch_epoch(it.epoch + 1)         # randperm of millions of rows costs ~20 ms: off the step path
        return self._step_staged(self._q_order[lo:lo + it.bs])

    def _q_prefetch_epoch(self, epoch: int):
        """build the NEXT epoch's permutation (same generator seeding as SeedIterator) on a host thread"""
        import threading
        it = self._q_iter

        def work():
            g = torch.Generator()
            g.manual_seed(it.seed * 1000003 + epoch)
            perm = torch.randperm(it.n, generator=g)
            self._q_next = (epoch, perm, self._q_vids[perm])
        self._q_thread = threading.Thread(target=work, daemon=True)
        self._q_thread.start()

    @property
    def epoch(self) -> int:
        return self._q_iter.epoch

    # ------------------------------------------------------------------ helpers
    def sample(self, seeds: torch.Tensor, out: Optional[List[torch.Tensor]] = None):
        """hop id lists [seeds, hop 1, ..., hop L]; with `out` (hop buffers, out[0] = seeds) hops 1..L are sampled
        into out[1:] (static buffers for graph capture)"""
        hops = [seeds]
        for i, k in enumerate(self.fanouts):
            nbr, _ = S.sample_neighbors(self.csr, hops[i], k, self.strategy, want_eids=False, rng=self.rng, salt=i + 1,
                                        out=None if out is None else out[i + 1])
            hops.append(nbr.reshape(-1) if out is None else out[i + 1])
        return hops

    # ------------------------------------------------------------------ what a subclass with other roots / loss replaces
    _fuse_ce = True         # the top layer's forward launch computes softmax-CE in its epilogue when it fits
    DROPOUT_SALT = 0x44524F50       # salt of the dropout seed ("DROP")
    BN_BUFFERS = ("running_mean", "running_var", "num_batches_tracked")

    def _fill_slot(self, slot: int, seed_ids_host: torch.Tensor):
        """write one host batch into pinned staging slot `slot` (here: B seed vids)"""
        self._h_seeds2[slot].copy_(seed_ids_host)

    def _put_roots(self, roots: torch.Tensor, seeds: torch.Tensor):
        """write a device batch into a root buffer (here: B seed vids)"""
        self.C.copy_i64(roots, seeds)

    def _stage(self, roots: torch.Tensor, host_slot: int):
        """captured head of the sampling branch: the staged batch (pinned slot, UVA-mapped) -> root buffer"""
        self.C.copy_i64(roots, self._h_seeds_dev[host_slot])

    def _draw_roots(self, roots: torch.Tensor):
        """complete a root buffer whose staged part is in place, before its hops are sampled (here: nothing)"""

    def _top_loss(self, seeds: torch.Tensor):
        """loss, dZ_L and the top bias gradient from the fp32 top-layer output when it was not fused"""
        top = self.layers[-1]
        self.C.softmax_ce(top.H, self.nodes.labels.local, seeds, self.rt.world, self.loss, top.dZ, top.db)

    # ------------------------------------------------------------------ the step
    def _step_body(self, pipe=None):
        """One training step as a small DAG of launches.  Independent work runs on forked streams (graph
        branches under capture) so that kernel-boundary latencies overlap instead of adding up:
            sampling: on main (plain schedule) or, under graph capture, the NEXT batch on its own branch, followed by
                      the rng + optimiser step counters
            main    : one persistent launch per layer (all hop pairs of the layer; the top layer also computes the loss)
            side A  : dW_L GEMM   ||   main : dA_L (sage_bwd_da) -> dW_{L-1} (dZ computed on the fly) -> dA_{L-1} ...
        everything joins before ONE fused kernel: gradient all-reduce + Adam + grad zeroing + next step's weight images."""
        C = self.C
        main = torch.cuda.current_stream()
        sA = self._side
        host_slot = None
        # no head work: the gradients were zeroed and the bf16 weight images refreshed by the fused Adam kernel of
        # the previous step (``repack()`` covers the very first step and externally modified weights)
        if pipe is None:
            # plain schedule: sample this step's batch, then train on it
            seeds = self.seeds
            self._draw_roots(seeds)
            hops = self.sample(seeds)
            # counters advance once the sampling kernels have consumed the RNG offset; needed again only by Adam
            self.opt.advance(self.rng.state)
        else:
            # pipelined schedule (graph capture): train on the batch sampled by the PREVIOUS replay while a
            # forked branch stages + samples the NEXT batch (the reference's sampling || training pipeline:
            # dag_scheduler.cc:51-62 / dag_dataset.cc:38-43, here inside one CUDA graph)
            cur, nxt, host_slot = pipe
            hops = self._hops[cur]
            seeds = hops[0]
            sS = self._sample_stream
            sS.wait_stream(main)
            with torch.cuda.stream(sS):
                if host_slot is not None:
                    # zero-copy staging: a tiny copy KERNEL reads the UVA-mapped pinned buffer over PCIe
                    self._stage(self._hops[nxt][0], host_slot)
                self._draw_roots(self._hops[nxt][0])
                self.sample(self._hops[nxt][0], out=self._hops[nxt])
                self.opt.advance(self.rng.state)
        # ---- forward: ONE persistent launch per layer covering all of its hop-pair segments; the top layer's
        # launch also computes the loss, dlogits and the bias gradient in its epilogue (fused CE)
        for ly in self.layers:
            if ly.below is None:    # self / neighbour rows: ids of hops i / i + 1 in the feature (or learned input) table
                d, self_ids, nbr_ids = self._input_desc(), hops[:ly.nseg], hops[1:ly.nseg + 1]
            else:                   # ... the contiguous row ranges of segments i / i + 1 of the layer below
                d, self_ids, nbr_ids = ly.below, [None] * ly.nseg, [None] * ly.nseg
            ce = [self.nodes.labels.local, seeds, self.loss, ly.dZ, ly.db] if ly.fuse_ce else []
            act = not ly.last and ly.bn is None         # ReLU + bf16 store in the epilogue; fp32 Z under batch norm
            if ly.split:                                # split-K: the self half's partial first
                C.sage_fused_multi(d, d, self_ids, [None] * ly.nseg, *ly.fwd_self, ly.mode, ly.img, None, ly.N, ly.n_out,
                                   False, False, [], self.rt.world, ly.ns, split_half=1)
            C.sage_fused_multi(d, d, self_ids, nbr_ids, *ly.fwd, ly.mode, ly.img, ly.conv.bias, ly.N, ly.n_out,
                               act, act, ce, self.rt.world, ly.ns, ly.amax, *ly.drop,
                               **({"split_half": 2, "partial": ly.fwd_self[4]} if ly.split else {}))
            b = ly.bn
            if b is not None:
                # per-segment statistics (+ the running buffers), then H = dropout(relu(BN(Z))) in bf16
                m, n = b.norm, ly.conv.out_dim
                C.bn_fwd_stats(b.Z, n, ly.offs, b.tickets[0], b.mean, b.rstd, m.running_mean, m.running_var,
                               m.num_batches_tracked, m.eps, m.momentum)
                C.bn_fwd_apply(b.Z, n, ly.offs, b.mean, b.rstd, m.weight, m.bias, ly.H, *b.drop)
            if ly.last and not ly.fuse_ce:
                # wide / split top layer: the loss runs as its own kernel on the (padded) logits
                self._top_loss(seeds)
        if host_slot is not None:
            # end-to-end graph: the loss leaves for pinned host slot `cur` on a branch parallel to the backward
            self._loss_stream.wait_stream(main)
            with torch.cuda.stream(self._loss_stream):
                self._h_loss_dev[cur].copy_(self.loss)
        # ---- backward: all GEMMs on wgmma (csrc/sage_bwd.cu), no library kernels
        #   top layer   : dW_L = dZ_L^T A_L with the dense dZ_L written by the fused loss epilogue
        #   layer l < L : dW_l = dZ_l^T A_l where dZ_l = relu'(H_l) * (self + 1/k neighbour rows of dA_{l+1}) is
        #                 computed inside the GEMM's producer warps (never stored for l = 1); bias grads fall out
        #                 (the scales and the argmax routing of the layer above's aggregator are in ly.bwd)
        #   dA_l = dZ_l . W_l  (l >= 2) on sage_bwd_da (mma.sync) over the layer's forward weight images, times
        #                 1 / (1 - p) when H_{l-1} is dropped out (dZ_l itself stays unscaled: dW_l reads it too)
        #   batch norm  : dY_l (routed as dZ_l above, into bn.dY) -> per-segment sum(dY), sum(dY x^) (+ d gamma, d beta)
        #                 -> dZ_l = gamma rstd (dY - mean(dY) - x^ mean(dY x^)), then dW_l on the dense dZ path beside dA_l
        for ly in reversed(self.layers):
            b = ly.bn
            if b is not None:
                m, n = b.norm, ly.conv.out_dim
                C.sage_bwd_dw(None, ly.H, a=None, dw=None, dbias=None, n_out=n, **ly.bwd)
                C.bn_bwd_reduce(b.dY, b.Z, n, ly.offs, b.tickets[1], b.mean, b.rstd, b.gsum, m.weight.grad, m.bias.grad)
                C.bn_bwd_apply(b.dY, b.Z, n, ly.offs, b.mean, b.rstd, m.weight, b.gsum, ly.dZ)
            if ly.last or b is not None:
                sA.wait_stream(main)
                with torch.cuda.stream(sA):            # dW_l runs beside dA_l
                    C.sage_bwd_dw(ly.dZ, None, [], [], [], [], [], [], 0, None, ly.A, ly.dW, None, ly.conv.out_dim)
            else:
                C.sage_bwd_dw(None, ly.H, a=ly.A, dw=ly.dW, dbias=ly.db, n_out=ly.conv.out_dim, **ly.bwd)
            if ly.dA is not None:
                # dA_l [rows, K_total] = dZ_l [rows, n_split * n_img] . W_l
                C.sage_bwd_da(ly.dZp, ly.img, ly.N, ly.ns, ly.dA, ly.da_alpha, ly.da_blocks)
        e = self.emb
        if e is not None:
            # dA_1 -> the gradient rows of the hop ids layer 1 read (+ their bits in the touched-row bitmap)
            ly = self.layers[0]
            C.embed_grad_scatter(ly.dA, self_ids=hops[:ly.nseg], nbr_ids=hops[1:ly.nseg + 1], grad=e.grad, bits=e.bits,
                                 **e.scatter)
        # ---- join, gradient all-reduce + fused optimiser (Adam + zero grads + next step's weight images)
        main.wait_stream(sA)
        if pipe is not None:
            main.wait_stream(self._sample_stream)
        if host_slot is not None:
            main.wait_stream(self._loss_stream)        # the loss must have left before the optimiser clears it
        o, ar = self.opt, self.ar
        if self._skip_opt:
            ar(self.flat_g, average=True)
            return
        if e is not None:
            # lazy Adam of the touched rows of E beside the dense optimiser, at the step count it uses (advanced above)
            sA.wait_stream(main)
            with torch.cuda.stream(sA):
                C.embed_lazy_adam(e.master, e.m, e.v, e.grad, e.table.local, e.bits, o.step_t, e.lr, o.betas[0],
                                  o.betas[1], o.eps)
        if ar.backend == "peer":
            # ONE kernel: stage grads (scaled, optionally bf16) -> cross-GPU flag barrier -> pull + reduce every peer's
            # slice in registers -> Adam -> zero grads -> next step's weight images (K8 fused with cast/scale + optimiser)
            C.adam_pack(self.flat_p, self.g_store, o.m, o.v, o.step_t, o.lr, o.betas[0], o.betas[1], o.eps, o.wd,
                        self.loss_out, self._mats, ar.desc, ar.epochs, ar.error, 1.0 / self.rt.world, self.ar_bf16,
                        self._drop_ctr)
        else:
            ar(self.flat_g, average=True)
            C.adam_pack(self.flat_p, self.g_store, o.m, o.v, o.step_t, o.lr, o.betas[0], o.betas[1], o.eps, o.wd,
                        self.loss_out, self._mats, None, None, None, 1.0, False, self._drop_ctr)
        if e is not None:
            main.wait_stream(sA)                        # E is updated before the next step's layer-1 forward reads it

    def repack(self):
        """Rebuild the bf16 weight images from the fp32 master weights (after init / load_state_dict / any
        external modification of the parameters)."""
        for ly in self.layers:
            ly.img.copy_(sage_ops.pack_images(ly.conv.weight_p, ly.N, ly.ns))

    # ------------------------------------------------------------------ graph / public step (same API as SageTrainer)
    def capture(self, warmup: int = 3):
        """Warm up eagerly, then capture four graphs (device-only pair + end-to-end pair, one per hop-buffer
        parity); the whole public ``step()`` - H2D of the seeds, sampling, training, D2H of the loss - is then
        ONE graph launch."""
        if not self.use_graph or self.graph is not None:
            return
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._step_body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.rt.barrier()
        # Four graphs over one memory pool, all software pipelined: graph i trains on hop buffers i and
        # samples the next batch into hop buffers i^1 on a forked branch.
        #   device-only pair : next seeds = whatever hop buffer i^1 holds (re-sampled with a fresh RNG offset)
        #   end-to-end pair  : + next seeds copied from pinned host slot i^1 at the head of the sampling branch
        #                      + loss -> pinned host slot i forked right after the loss kernel
        # No PCIe round trip and no sampling kernel sits on the critical path (tools/diag_e2e.py).
        self._sample_stream = torch.cuda.Stream(priority=0)
        cap_stream = torch.cuda.Stream(priority=-1)
        self._hops = [[torch.zeros(n, dtype=torch.int64, device=self.rt.device) for n in self.n] for _ in range(2)]
        self._hops[0][0] = self.seeds                      # `tr.seeds` stays the handle of buffer 0
        self._seeds_bufs = [self._hops[0][0], self._hops[1][0]]
        self._prime_hops(0)
        self._dev_graphs, self._e2e_graphs = [], []
        pool = None
        for e2e in (False, True):
            for i in range(2):
                gi = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gi, pool=pool, stream=cap_stream):
                    self._step_body(pipe=(i, i ^ 1, (i ^ 1) if e2e else None))
                pool = gi.pool() if pool is None else pool
                (self._e2e_graphs if e2e else self._dev_graphs).append(gi)
        self.graph = self._dev_graphs[0]
        self._primed = False
        torch.cuda.synchronize()
        self.rt.barrier()

    def _prime_hops(self, i: int):
        """Sample the roots in hop buffer i into it and copy the batch to buffer i^1, so that whichever graph replays
        first finds a batch."""
        self._draw_roots(self._hops[i][0])
        self.sample(self._hops[i][0], out=self._hops[i])
        for dst, src in zip(self._hops[i ^ 1], self._hops[i]):
            dst.copy_(src)

    def step_device(self, next_seeds: Optional[torch.Tensor] = None):
        """Device-only step (no host traffic): graph replay on the resident seed buffers.  ``next_seeds`` (device
        int64 [B]) are the seeds of the batch the replay samples for the FOLLOWING step (software pipeline); without
        them the resident seeds are re-sampled with a fresh RNG offset."""
        self._step_device(next_seeds)

    def _step_device(self, *next_roots):
        """``step_device`` of any root layout: `next_roots` are ``_put_roots``'s arguments, or start with None when
        the step has no new roots"""
        if self.graph is not None:
            i = self._steps & 1
            if next_roots[0] is not None:
                self._put_roots(self._hops[i ^ 1][0], *next_roots)
                if not self._primed:
                    self._put_roots(self._hops[i][0], *next_roots)
            if not self._primed:
                self._prime_hops(i)
                self._primed = True
            self._dev_graphs[i].replay()
        else:
            if next_roots[0] is not None:
                self._put_roots(self.seeds, *next_roots)
            self._step_body()
        self._steps += 1

    def step(self, seed_ids_host: torch.Tensor) -> torch.Tensor:
        """End-to-end step through the public path: host seed ids -> (pinned staging) -> device,
        train, loss -> pinned host.  Asynchronous: synchronise before reading the returned tensor.
        With CUDA graphs the copies are nodes of the step graph (double-buffered staging)."""
        return self._step_staged(seed_ids_host)

    def _step_staged(self, *batch) -> torch.Tensor:
        """``step`` of any root layout: `batch` are ``_fill_slot``'s arguments.  Call t fills pinned staging slot
        (t & 1) ^ 1 and returns pinned loss slot t & 1.  Eagerly it trains on its own batch.  With CUDA graphs it is
        pipelined: the batch is copied to the device inside the graph, in parallel with the training step, which
        trains on the batch staged by the PREVIOUS call (the very first call also places its batch directly)."""
        i = self._steps & 1
        self._e2e_done[i].synchronize()        # step t-2 was the last reader of staging slot i^1
        self._fill_slot(i ^ 1, *batch)
        if self.graph is None:
            self._stage(self.seeds, i ^ 1)
            self._step_body()
            self._h_loss2[i].copy_(self.loss_out, non_blocking=True)
        else:
            if not self._primed:
                self._stage(self._hops[i][0], i ^ 1)
                self._prime_hops(i)
                self._primed = True
            self._e2e_graphs[i].replay()
        self._e2e_done[i].record()
        self._steps += 1
        self.h_loss = self._h_loss2[i]
        return self.h_loss

    def synchronize(self):
        torch.cuda.synchronize()

    @torch.no_grad()
    def predict(self, seeds: torch.Tensor) -> torch.Tensor:
        self.model.eval()
        hops = self.sample(seeds)
        out = self.model.forward_store(self.nodes if self.emb is None else self.emb.view, hops, self.fanouts)
        self.model.train()
        return out

    @torch.no_grad()
    def infer_all(self) -> torch.Tensor:
        """Layer-wise full-neighbourhood forward of the trained model: fp32 ``[n_local, out_dim]`` for every local node
        of the node table, row r = the node with vid ``r * world + rank`` (logits of a supervised trainer, embeddings of
        a link trainer).  Layer l aggregates the FULL adjacency row of every node in ``self.csr`` (the neighbourhood
        training samples from) over the outputs of layer l - 1: one fused launch per layer, plus one hub pre-pass
        launch per layer when the CSR has rows above ``ops.sage.CSR_HUB_DEGREE``.  It uses the resident weight images
        and the training forward's layer semantics (hidden layers ReLU -> bf16, top layer fp32; batch norm in eval mode, with
        the running statistics, folded into the weights and bias), is deterministic and is
        the expectation that the sampled ``predict`` estimates.  Training state is not touched.  Collective when
        world > 1 (the hidden-layer tables are symmetric, allocated on the first call).  Export::

            from graphlearn_b200.utils.checkpoint import save_embeddings
            ids = tr.nodes.idmap.to_id(tr.nodes.idmap.local_vids())
            save_embeddings(path, ids, tr.infer_all())
        """
        from ..parallel.runtime import make_table_desc
        rt, n = self.rt, self.nodes.n_local
        if self._inf is None:
            plan = sage_ops.CsrPlan(self.csr.indptr.local, self.csr.indices.local, n)
            tabs = []
            for c in self.convs[:-1]:
                stride = (c.out_dim + 7) // 8 * 8                  # 16-byte bf16 rows
                st = rt.symm_empty((n, stride), torch.bfloat16)
                tabs.append((st, make_table_desc(rt.world, c.out_dim, stride, torch.bfloat16, st.nrows, st.ptrs)))
            rt.barrier()
            self._inf = (plan, self.nodes.idmap.local_vids(), tabs)
        plan, vids, tabs = self._inf
        rt.barrier()                                                # peers are done reading the previous call's tables
        desc = self._input_desc()
        for l, ly in enumerate(self.layers):
            c = ly.conv
            if ly.last:                                             # image i writes columns [i n_out, i n_out + n_out)
                res = torch.empty(n, ly.ns * ly.n_out, dtype=torch.float32, device=rt.device)
                out = res[:, :ly.n_out]
            else:
                out = tabs[l][0].local[:, :ly.n_out]
            img, bias = ly.img, c.bias
            if ly.bn is not None:
                # eval-mode BN folded into the layer: s = gamma / sqrt(running_var + eps), W' = diag(s) W,
                # b' = beta - s running_mean (inference-only images: ly.img belongs to the optimiser)
                m = ly.bn.norm
                s = m.weight / torch.sqrt(m.running_var + m.eps)
                img = sage_ops.pack_images(c.weight_p * s[:, None], ly.N, ly.ns)
                bias = (m.bias - s * m.running_mean).contiguous()
            plan.layer(desc, desc, vids, out, c.agg_type, img, bias, ly.N, ly.n_out, not ly.last, not ly.last, ly.ns,
                       split_k=ly.split)
            if not ly.last:
                desc = tabs[l][1]
                rt.barrier()                                        # layer l + 1 reads peer rows of layer l
        return res[:, :c.out_dim]

    @torch.no_grad()
    def evaluate(self, vids: torch.Tensor) -> float:
        """Accuracy of the argmax of the ``infer_all()`` rows of the local nodes `vids` (device int64) against the node
        table's labels (supervised trainers)."""
        rows = torch.div(vids, self.rt.world, rounding_mode="floor")
        pred = self.infer_all()[rows].argmax(1)
        return float((pred == self.nodes.labels.local[rows]).float().mean())

    def state_dict(self):
        sd = {"model": self.flat_p.clone(), "opt": self.opt.state_dict(), "rng": self.rng.state_dict(),
              "steps": self._steps, "dropout_state": self.drop_state.cpu()}
        if self.emb is not None:
            sd["input_embedding"] = {"master": self.emb.master.clone(), "m": self.emb.m.clone(), "v": self.emb.v.clone()}
        if self.batch_norm:
            sd["batch_norm"] = [{k: getattr(ly.bn.norm, k).clone() for k in self.BN_BUFFERS} for ly in self.layers[:-1]]
        return sd

    def load_state_dict(self, sd):
        if self.emb is not None and "input_embedding" not in sd:
            raise ValueError("the checkpoint has no learned input embedding, which this trainer trains")
        if self.batch_norm and len(sd.get("batch_norm", ())) != self.L - 1:
            raise ValueError("the checkpoint has no batch-norm running statistics for the %d hidden layers this trainer "
                             "normalises" % (self.L - 1))
        self.flat_p.copy_(sd["model"])
        self.repack()
        self.opt.load_state_dict(sd["opt"])
        self.rng.load_state_dict(sd["rng"])
        self._steps = int(sd["steps"])
        if "dropout_state" in sd:       # (checkpoints written before dropout training keep this trainer's own state)
            self.drop_state.copy_(sd["dropout_state"])
        if self.emb is not None:
            e, s = self.emb, sd["input_embedding"]
            e.master.copy_(s["master"]); e.m.copy_(s["m"]); e.v.copy_(s["v"])
            e.table.local[:, :e.master.size(1)] = e.master.to(torch.bfloat16)
        if self.batch_norm:
            for ly, st in zip(self.layers[:-1], sd["batch_norm"]):
                for k in self.BN_BUFFERS:
                    getattr(ly.bn.norm, k).copy_(st[k])
