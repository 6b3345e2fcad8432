"""Multi-GPU plumbing: nodes-to-explain are independent units, so they are dealt across ranks (one process per GPU) with
NO data-path collective; the only exchange is ONE all-gather of the packed edge masks at the end.

How one collective suffices: every rank knows the k-hop subgraph size of EVERY node of the list (gx_count_nodes: the
integer frontier expansion without building a plan, remembered per graph), so the shard assignment (cost balanced), every
rank's payload size and every item's offset are known everywhere without a metadata exchange.  Each rank pads its packed masks to
the largest per-rank payload, ONE all-gather moves the slots (NCCL over NVLink through the library's own communicator,
gx_allgather_masks; torch.distributed -- gloo in the CPU tests -- when no engine communicator exists), and a device kernel
(gx_unshard_masks) scatters the slots into input order.  The masks never leave the device between the explainer kernels and
the collective.

Per-node arithmetic never crosses a GPU, so results are bit-identical to the 1-GPU run (tests/test_gpu_dist.py,
tests/test_dist_gloo.py, bench.py "shard_bit_identical").

Graph-classification mode is dealt the same way, graph by graph (explain_graphs_sharded): gx_count_graphs gives every graph's payload
from the batch CSR on the host, and gx_densify_graphs turns the gathered masks into explain_graphs' dense arrays on device
(tests/test_gpu_dist_graphs.py, tests/test_gpu_dist_graphs_multi.py).

Graphs whose full masks cannot be gathered (BASELINE configs[4]) deliver denoise_graph's top-k edges instead (explain_nodes_topk_sharded):
each rank explains its share a chunk at a time and keeps the thresholded edges in global node ids on device (gx_denoise_topk_edges); two
all-gathers move (threshold, count) per node and 3 words per edge (allgather_topk; tests/test_gpu_topk_edges.py, test_topk_gather_gloo.py)."""
import numpy as np
import torch
import torch.distributed as dist

from .explain import _m0_at_edges, torch_m0_walk


def shard_indices(num_items, world, rank, costs=None):
    """Positions (into the caller's node list) owned by `rank`.  With costs: sort by cost
    descending and deal round-robin (LPT-style balance); otherwise plain round-robin."""
    if costs is None:
        order = np.arange(num_items)
    else:
        order = np.argsort(-np.asarray(costs), kind="stable")
    return np.sort(order[rank::world])


def shard_layout(sizes_all, world, costs=None):
    """Everything a rank needs to know about the exchange, computed identically on every rank from the per-item sizes:
    shards[r] = positions of rank r; slot = floats per rank in the all-gather (largest payload); src_off[p] = where item p sits in
    the gathered [world*slot] buffer; offsets[p] = where it goes in input order."""
    sizes_all = np.asarray(sizes_all, np.int64)
    num = len(sizes_all)
    order = np.argsort(-np.asarray(sizes_all if costs is None else costs), kind="stable")     # one sort; shard r = every world-th item of it
    shards = [np.sort(order[r::world]) for r in range(world)]
    slot = max(1, max(int(sizes_all[s].sum()) for s in shards))
    offsets = np.concatenate([[0], np.cumsum(sizes_all)]).astype(np.int64)
    src_off = np.zeros(num, np.int64)
    for r, s in enumerate(shards):
        if len(s):
            src_off[s] = r * slot + np.concatenate([[0], np.cumsum(sizes_all[s])[:-1]])
    return shards, slot, src_off, offsets


def allgather_packed(local_vals, sizes_all, rank, world, costs=None, group=None, engine=None, out=None, layout=None):
    """ONE all-gather of ragged per-item float32 payloads.
    local_vals : 1-D float32 tensor = this rank's items (positions shard_layout(...)[0][rank], ascending) concatenated
    sizes_all  : payload length of EVERY item of the list (known on every rank: gx_count_nodes)
    Returns (values, offsets): all payloads concatenated in input order, int64 offsets[num_items+1]."""
    shards, slot, src_off, offsets = layout if layout is not None else shard_layout(sizes_all, world, costs)
    sizes_all = np.asarray(sizes_all, np.int64)
    device = local_vals.device
    total = int(offsets[-1])
    assert local_vals.numel() == int(sizes_all[shards[rank]].sum()), "local payload does not match the shard layout"
    if engine is not None and getattr(engine, "comm_world", None) == world and device.type == "cuda":
        gathered = engine.allgather_masks(local_vals.contiguous(), slot)                 # gx_allgather_masks: one ncclAllGather
        values = out if out is not None else torch.empty(max(total, 1), dtype=torch.float32, device=device)
        engine.unshard_masks(gathered, src_off, offsets[:-1], sizes_all, values)         # gx_unshard_masks: device scatter
        return values[:total], offsets
    pay = torch.zeros(slot, dtype=torch.float32, device=device)
    pay[: local_vals.numel()] = local_vals
    gathered = torch.empty(world * slot, dtype=torch.float32, device=device)
    dist.all_gather_into_tensor(gathered, pay, group=group)                               # THE collective (gloo / torch's NCCL)
    item_of = np.repeat(np.arange(len(sizes_all)), sizes_all)
    idx = torch.from_numpy(src_off[item_of] + (np.arange(total) - offsets[:-1][item_of])).to(device)
    return gathered[idx], offsets


def ensure_comm(engine, group=None):
    """Bootstraps the engine's own NCCL communicator (gx_comm_init) once per process group: rank 0 creates the id, one
    broadcast_object_list transports it."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if getattr(engine, "comm_world", None) == world:
        return
    box = [engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0, group=group)
    engine.comm_init(world, rank, box[0])


def count_nodes_cached(explainer, nodes):
    """(n, E_d) of every node of the list.  The k-hop sizes are a property of (graph, node, n_hops), so they are counted once per
    Explainer graph (gx_count_nodes on the nodes not seen yet) and remembered: a steady stream of explain calls pays nothing here."""
    eng = explainer.engine
    key = (getattr(explainer, "_current_graph", 0), int(explainer.n_hops))
    cache = explainer.__dict__.setdefault("_count_cache", {})
    if key not in cache:
        N = eng.num_nodes
        cache[key] = (np.full(N, -1, np.int64), np.zeros(N, np.int64))
    n_c, e_c = cache[key]
    nodes = np.asarray(nodes, np.int64)
    todo = np.unique(nodes[n_c[nodes] < 0])
    if len(todo):
        n_new, e_new = eng.count_nodes(todo.astype(np.int32), explainer.n_hops)
        n_c[todo] = n_new; e_c[todo] = e_new
    return n_c[nodes], e_c[nodes]


def explain_nodes_sharded(explainer, node_indices, costs=None, group=None, use_engine_comm=True):
    """Explainer.explain_nodes across all ranks of the default process group.
    Every rank returns the packed masks of ALL nodes: (values float32 tensor, offsets int64 array, (local plan or None, local positions));
    values[offsets[t]:offsets[t+1]] are the masked_adj entries of node_indices[t] at the row-major sub-adjacency slots."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    eng = explainer.engine
    eng.follow_torch_stream()
    nodes = np.asarray(node_indices)
    dev = torch.device("cuda", eng.device)
    n_all, e_all = count_nodes_cached(explainer, nodes)
    # the layout of a node list is a pure function of (list, world, costs): remembered for the list that was explained last
    key = (nodes.tobytes(), world, None if costs is None else np.asarray(costs).tobytes(), getattr(explainer, "_current_graph", 0))
    memo = explainer.__dict__.get("_layout_memo")
    if memo is None or memo[0] != key:
        memo = (key, shard_layout(e_all, world, costs))
        explainer._layout_memo = memo
    layout = memo[1]
    pos = layout[0][rank]
    hp, init = explainer._hparams()
    if len(pos):
        # the canonical sub-graph description comes back to the host only when the torch-compatible init needs it (M0 gather)
        plan = eng.plan_nodes(nodes[pos], explainer.n_hops, fetch=(init == "torch"))
        m0_dev = None
        if init == "torch":   # every rank walks the whole list so that torch's RNG is consumed exactly as one process would
            mine = set(pos.tolist())
            walk = enumerate(torch_m0_walk(n_all))
            m0_dev = torch.from_numpy(_m0_at_edges(plan, (M for p, M in walk if p in mine))).to(dev)
            for _ in walk:
                pass
        local = eng.explain_nodes_device(hp, m0_dev)
    else:
        plan, local = None, torch.zeros(0, dtype=torch.float32, device=dev)
    if use_engine_comm:
        ensure_comm(eng, group)
    values, offsets = allgather_packed(local, e_all, rank, world, costs, group=group, engine=eng if use_engine_comm else None, layout=layout)
    return values, offsets, (plan, pos)


def explain_graphs_sharded(explainer, graph_indices, costs=None, group=None, use_engine_comm=True, dense=False, model="exp"):
    """Explainer(graph_mode=True).explain_graphs across all ranks of the default process group (or `group`): each rank explains its
    share of the graph list, ONE all-gather delivers every graph's packed masks.  Every model and optimiser explain_graphs accepts.
    costs: per-graph cost for the balance (default: the graph's directed edges, gx_count_graphs).  The layout is remembered for the list
    explained last, like explain_nodes_sharded's.
    Every rank returns (values float32 CUDA tensor, offsets int64 array, (edge_off of this rank's plan or None, this rank's positions));
    values[offsets[t]:offsets[t+1]] are the masked_adj entries of graph_indices[t] at its CSR slots (row-major).  dense=True appends the
    (len(graph_indices), max_nodes, max_nodes) float64 CUDA tensor of the dense arrays explain_graphs returns (gx_densify_graphs).
    With args.gnnx_init = "torch" every rank draws the n^2 normals of EVERY graph of the list (torch's RNG ends as after one process's
    explain_graphs); "device" draws nothing on the host.  Unlike explain_graphs it prints no per-epoch trace and writes no .npy files.
    model="grad": the gradient baseline of every graph (explain_graphs(model="grad")), dealt, gathered and densified the same way."""
    if not explainer.graph_mode:
        raise ValueError("explain_graphs_sharded needs an Explainer constructed with graph_mode=True")
    if model not in ("exp", "grad"):
        raise NotImplementedError("model=%r is not built in graph mode" % model)
    if model == "grad":
        explainer._check_graph_grad()     # before any RNG is consumed
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    eng = explainer.engine
    eng.follow_torch_stream()
    gids = np.asarray(graph_indices, np.int64)
    dev = torch.device("cuda", eng.device)
    key = (gids.tobytes(), world, None if costs is None else np.asarray(costs).tobytes())
    memo = explainer.__dict__.get("_graph_layout_memo")
    if memo is None or memo[0] != key:
        _, e_all = eng.count_graphs(gids)
        memo = (key, e_all, shard_layout(e_all, world, costs))
        explainer._graph_layout_memo = memo
    _, e_all, layout = memo
    pos = layout[0][rank]
    hp, init = explainer._hparams()
    m0_host = None
    if init == "torch":   # every rank walks the whole list, owning graphs or not, so that torch's RNG is consumed as one process would
        m0_host = explainer._draw_graph_m0_subset(eng.batch_n, len(gids), pos, [eng.graph_rows_cols(int(g)) for g in gids[pos]])
    if len(pos):
        edge_off = eng.plan_graphs(gids[pos])
        if model == "grad":
            local = eng.grad_graphs_device(explainer._graph_grad_labels(gids[pos]))
        else:
            local = eng.explain_graphs_device(hp, None if m0_host is None else torch.from_numpy(m0_host).to(dev))
    else:
        edge_off, local = None, torch.zeros(0, dtype=torch.float32, device=dev)
    if use_engine_comm:
        ensure_comm(eng, group)
    values, offsets = allgather_packed(local, e_all, rank, world, costs, group=group, engine=eng if use_engine_comm else None, layout=layout)
    if dense:
        return values, offsets, (edge_off, pos), eng.densify_graphs_device(gids, values)
    return values, offsets, (edge_off, pos)


def explain_nodes_topk_sharded(explainer, node_indices, threshold_num=20, chunk_size=None, costs=None, group=None, use_engine_comm=True,
                               timings=None):
    """Explainer.explain_nodes_topk across all ranks of the default process group (or `group`), for lists whose full masks cannot be
    gathered (BASELINE configs[4]: 3.4 GB of masks per 132 nodes).  The nodes are dealt as in explain_nodes_sharded (count_nodes_cached,
    shard_layout, cost = E_d unless `costs`); each rank runs explain_nodes_topk's chunk loop over its own positions, then TWO all-gathers
    (allgather_packed: gx_allgather_masks / gx_unshard_masks with the engine's communicator, torch.distributed without it) deliver
      1. (threshold, count) of every node -- 2 words each, sizes known in advance;
      2. the kept edges -- 3 words each: u and v bit-cast int32, then the value; the sizes come from gather 1, and the layout keeps the
         explanation's shards (the same costs, no re-sort by record size).
    Every rank returns (thr, offsets, uv, vals, positions): thr / offsets / uv / vals exactly as explain_nodes_topk(node_indices) on one
    GPU, bit for bit; positions = the list entries this rank explained.  With args.gnnx_init = "torch" every rank walks the whole list
    through torch's RNG once, keeping the normals of its own nodes chunk by chunk.
    timings (dict or None): per-rank wall seconds of count, plan, m0, explain, topk, gather1, gather2 (synchronising after each phase),
    the explainer kernels' device seconds (explain_device) and the gathered bytes."""
    import time
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    eng = explainer.engine
    if explainer.graph_mode:
        raise ValueError("explain_nodes_topk_sharded is node mode only")
    eng.follow_torch_stream()
    nodes = np.asarray(node_indices, np.int64).reshape(-1)
    dev = torch.device("cuda", eng.device)
    t0 = time.perf_counter()
    n_all, e_all = count_nodes_cached(explainer, nodes)
    cost = np.asarray(e_all if costs is None else costs)
    shards = shard_layout(e_all, world, cost)[0]
    pos = shards[rank]
    if timings is not None:
        timings["count"] = timings.get("count", 0.0) + time.perf_counter() - t0
    thr, cnt, uv, vals = explainer._topk_chunks(nodes, pos, n_all, threshold_num, chunk_size, timings=timings)
    if use_engine_comm:
        ensure_comm(eng, group)
    thr, offsets, uv, vals = allgather_topk(thr, cnt, uv, vals, cost, group=group, engine=eng if use_engine_comm else None, timings=timings)
    return thr, offsets, uv, vals, pos


def allgather_topk(thr, counts, uv, vals, costs, group=None, engine=None, timings=None):
    """The two all-gathers of explain_nodes_topk_sharded.  This rank's items are the positions shard_layout(costs, world, costs)[0][rank]
    (ascending) of a list of len(costs) items: thr [k] float32 and counts [k] (host) per item, and the items' records uv [sum counts, 2]
    int32 and vals [sum counts] float32, item after item (tensors on one device).  Gather 1 moves (threshold, count) of every item, 2 words
    each; gather 2 moves 3 words per record (u, v bit-cast, value) with sizes from gather 1, in the same shards (layouts from `costs`, not
    from the record sizes).  Both go through allgather_packed (engine: the library's communicator).
    Returns (thr [num], offsets int64 [num+1], uv [total, 2], vals [total]) of the whole list in list order, on every rank."""
    import time
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    costs = np.asarray(costs)
    num = len(costs)
    dev = thr.device

    def gathered(key, local, sizes):
        t1 = time.perf_counter()
        out, _ = allgather_packed(local, sizes, rank, world, group=group, engine=engine, layout=shard_layout(sizes, world, costs))
        if timings is not None:
            if dev.type == "cuda":
                torch.cuda.synchronize(dev)
            timings[key] = timings.get(key, 0.0) + time.perf_counter() - t1
            timings[key + "_bytes"] = timings.get(key + "_bytes", 0) + 4 * int(np.sum(sizes))
        return out

    # 1. (threshold, count) per item
    cnt32 = torch.from_numpy(np.ascontiguousarray(counts, np.int32)).to(dev)
    head = torch.stack([thr.float(), cnt32.view(torch.float32)], 1).reshape(-1)
    g1 = gathered("gather1", head, np.full(num, 2, np.int64)).view(-1, 2)
    cnt_all = g1[:, 1].contiguous().view(torch.int32).cpu().numpy().astype(np.int64)
    # 2. the records, in the same shards
    rec = torch.cat([uv.contiguous().view(torch.float32), vals.reshape(-1, 1)], 1).reshape(-1)
    g2 = gathered("gather2", rec, 3 * cnt_all).view(-1, 3)
    offsets = np.concatenate([[0], np.cumsum(cnt_all)]).astype(np.int64)
    return g1[:, 0].contiguous(), offsets, g2[:, :2].contiguous().view(torch.int32), g2[:, 2].contiguous()
