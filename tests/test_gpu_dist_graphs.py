"""GPU (-m gpu), one device: graph-classification mode sharded by graph (gnnx.dist.explain_graphs_sharded, gx_count_graphs,
gx_densify_graphs).

Rank emulation: for world sizes 1, 2, 3, 4 and 8 every rank's shard is planned and explained on its own, as explain_graphs_sharded does on
that rank, and the shards are put together with shard_layout on the host; the result must be explain_graphs on the whole list, bit for
bit -- the tuned kernel with the torch and the device init, a --bn 4-layer model with RMSprop and a step scheduler, attention and MLP-head
models, and a batch over several launch classes.  End to end: a one-rank group through explain_graphs_sharded(dense=True), with the
library's NCCL communicator and with torch.distributed (gloo)."""
import socket
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist

import gnnx
from gnnx import _abi
from gnnx import dist as gdist
import util
from test_gpu_graph_shapes import _ba, _batch, _classes_run

pytestmark = pytest.mark.gpu
GX_ERR_INVALID = -1
WORLDS = (1, 2, 3, 4, 8)


@pytest.fixture(scope="module")
def gg():
    return np.load(util.GOLDEN + "/graphs_golden.npz")


def _args(tmp_path, L=3, init="torch", **over):
    a = dict(num_gc_layers=L, num_epochs=20, lr=0.1, opt="adam", opt_scheduler="none", mask_act="sigmoid", mask_bias=False, gpu=False,
             bias=True, method="base", dataset="graphs", bmname=None, hidden_dim=20, output_dim=20, name_suffix="", explainer_suffix="",
             logdir=str(tmp_path), gnnx_init=init, gnnx_seed=11)
    a.update(over)
    return types.SimpleNamespace(**a)


def _explainer(adj, feat, label, args, L=3, bn=False, head=(), weights=None):
    """The drop-in Explainer in graph mode on a gnnx.models.GcnEncoderGraph (torch's init under a fixed seed, or `weights`)."""
    torch.manual_seed(17)
    C = int(np.max(label)) + 1 if weights is None else weights["Wp"].shape[0]
    model = gnnx.models.GcnEncoderGraph(feat.shape[2], 20, 20, max(C, 2), L, pred_hidden_dims=list(head), bn=bn, args=args)
    if weights is not None:
        sd = {"conv_first.weight": weights["W1"], "conv_first.bias": weights["b1"], "conv_block.0.weight": weights["W2"],
              "conv_block.0.bias": weights["b2"], "conv_last.weight": weights["W3"], "conv_last.bias": weights["b3"],
              "pred_model.weight": weights["Wp"], "pred_model.bias": weights["bp"]}
        model.load_state_dict({k: torch.tensor(np.asarray(v)) for k, v in sd.items()})
    return gnnx.Explainer(model=model, adj=torch.tensor(adj, dtype=torch.float), feat=torch.tensor(np.asarray(feat, np.float32)),
                          label=torch.tensor(np.asarray(label)), pred=None, train_idx=[], args=args, writer=None, print_training=False,
                          graph_mode=True, graph_idx=0)


def _emulated_rank(ex, gids, layout, rank):
    """What explain_graphs_sharded computes on `rank` before the gather: this rank's packed masks (host)."""
    eng = ex.engine
    pos = layout[0][rank]
    hp, init = ex._hparams()
    m0 = None
    if init == "torch":
        m0 = ex._draw_graph_m0_subset(eng.batch_n, len(gids), pos, [eng.graph_rows_cols(int(g)) for g in gids[pos]])
    if not len(pos):
        return np.zeros(0, np.float32)
    eng.plan_graphs(gids[pos])
    local = eng.explain_graphs_device(hp, None if m0 is None else torch.from_numpy(m0).cuda())
    return local.cpu().numpy()


def _check_rank_emulation(ex, gids, seed=3):
    """Every world size, every rank: the assembled shards == explain_graphs(gids), packed and densified, and torch's RNG ends alike."""
    gids = np.asarray(gids, np.int64)
    torch.manual_seed(seed)
    want = ex.explain_graphs(gids.tolist(), save=False)
    rng_after = torch.get_rng_state()
    eng = ex.engine
    want_packed = np.concatenate([D[eng.graph_rows_cols(int(g))] for D, g in zip(want, gids)]).astype(np.float32)
    _, e_all = eng.count_graphs(gids)
    for world in WORLDS:
        layout = gdist.shard_layout(e_all, world)
        shards, slot, src_off, offsets = layout
        gathered = np.zeros(world * slot, np.float32)
        for rank in range(world):
            torch.manual_seed(seed)
            local = _emulated_rank(ex, gids, layout, rank)
            assert torch.equal(torch.get_rng_state(), rng_after), (world, rank)
            gathered[rank * slot: rank * slot + len(local)] = local
        values = np.concatenate([gathered[src_off[p]: src_off[p] + e_all[p]] for p in range(len(gids))])
        assert np.array_equal(values, want_packed, equal_nan=True), world
        dense = eng.densify_graphs_host(gids, values)
        assert all(np.array_equal(dense[t], want[t], equal_nan=True) for t in range(len(gids))), world
    return want


# ------------------------------------------------------------------------------------------------ rank emulation
@pytest.mark.parametrize("init", ["torch", "device"])
def test_rank_emulation_tuned_kernel(gg, tmp_path, init):
    ex = _explainer(gg["adj"], gg["feat"], gg["label"], _args(tmp_path, init=init), weights={k: gg[k] for k in util.WKEYS})
    _check_rank_emulation(ex, [3, 0, 11, 7, 7, 5, 1, 9, 2, 10, 4, 6, 8])      # a repeated graph, out of order
    ex.engine.close()


def test_rank_emulation_bn_4_layers_rmsprop_step(gg, tmp_path):
    args = _args(tmp_path, L=4, opt="rmsprop", opt_scheduler="step", opt_decay_step=7, opt_decay_rate=0.5)
    ex = _explainer(gg["adj"], gg["feat"], gg["label"], args, L=4, bn=True)
    _check_rank_emulation(ex, list(range(12)))
    ex.engine.close()


@pytest.mark.parametrize("kind", ["att", "head"])
def test_rank_emulation_attention_and_mlp_head(gg, tmp_path, kind):
    if kind == "att":
        ex = _explainer(gg["adj"], gg["feat"], gg["label"], _args(tmp_path, method="att"))
        assert ex._att
    else:
        ex = _explainer(gg["adj"], gg["feat"], gg["label"], _args(tmp_path, init="device"), bn=True, head=[50])
        assert ex._head
    _check_rank_emulation(ex, [11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1, 0])
    ex.engine.close()


def test_rank_emulation_across_launch_classes(tmp_path):
    rng = np.random.default_rng(8)
    sizes = [6, 15, 30, 50, 90, 12, 40, 8]
    n = 96
    adj = _batch([_ba(s, seed=s) for s in sizes], n)
    feat = rng.normal(size=(len(sizes), n, 14)).astype(np.float32) * (adj.sum(2, keepdims=True) > 0)
    ex = _explainer(adj, feat, rng.integers(0, 2, len(sizes)), _args(tmp_path))
    gids = list(range(len(sizes)))
    torch.manual_seed(0)
    ex.explain_graphs(gids, save=False)
    assert len(_classes_run(ex.engine)) >= 3, _classes_run(ex.engine)
    _check_rank_emulation(ex, gids)
    ex.engine.close()


# ------------------------------------------------------------------------------------------------ end to end, one rank
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def test_explain_graphs_sharded_one_rank(gg, tmp_path):
    gids = [4, 1, 9, 1, 0, 11, 6]
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % _free_port(), rank=0, world_size=1)
    try:
        ex = _explainer(gg["adj"], gg["feat"], gg["label"], _args(tmp_path), weights={k: gg[k] for k in util.WKEYS})
        torch.manual_seed(21)
        want = ex.explain_graphs(gids, save=False)
        rng_after = torch.get_rng_state()
        for use_engine_comm in (False, True):        # torch.distributed (gloo), then the library's NCCL communicator
            torch.manual_seed(21)
            values, offsets, (edge_off, pos), dense = gdist.explain_graphs_sharded(ex, gids, use_engine_comm=use_engine_comm, dense=True)
            assert torch.equal(torch.get_rng_state(), rng_after)
            assert dense.dtype == torch.float64 and dense.is_cuda and tuple(dense.shape) == (len(gids),) + want[0].shape
            dense = dense.cpu().numpy()
            assert all(np.array_equal(dense[t], want[t]) for t in range(len(gids))), use_engine_comm
            assert np.array_equal(pos, np.arange(len(gids))) and np.array_equal(edge_off, offsets)
            v = values.cpu().numpy()
            for t, g in enumerate(gids):
                assert np.array_equal(v[offsets[t]:offsets[t + 1]], want[t][ex.engine.graph_rows_cols(g)].astype(np.float32))
        assert not any(f.suffix == ".npy" for f in tmp_path.iterdir())       # no .npy side effect
        # the layout is remembered per (list, world, costs): a second call counts nothing
        calls = []
        count = ex.engine.count_graphs
        ex.engine.count_graphs = lambda g: (calls.append(1), count(g))[1]
        gdist.explain_graphs_sharded(ex, gids, use_engine_comm=False)
        assert not calls
        gdist.explain_graphs_sharded(ex, gids[:3], use_engine_comm=False)
        assert len(calls) == 1
        ex.engine.close()
    finally:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ gx_densify_graphs, gx_count_graphs
def _host_densify(eng, gids, values):
    """_explain_graph_batch's densify: D[rows, cols] = the graph's slots, graph after graph."""
    n, out, o = eng.batch_n, [], 0
    for g in gids:
        r, c = eng.graph_rows_cols(g)
        D = np.zeros((n, n), np.float64)
        D[r, c] = values[o:o + len(r)]
        out.append(D)
        o += len(r)
    return np.stack(out) if out else np.zeros((0, n, n))


@pytest.mark.parametrize("n", [40, 33])
def test_densify_graphs_host_and_device(gg, n):
    """Host and device buffers against the host densify; n = 33 puts every other graph's block at an odd double (a scalar head store)."""
    eng = gnnx.Engine(0)
    adj = np.zeros((12, n, n), np.uint8)
    m = min(n, 40)
    adj[:, :m, :m] = gg["adj"][:, :m, :m]
    eng.set_graph_batch(adj, np.zeros((12, n, 1), np.float32), gg["label"])
    gids = [5, 0, 11, 5, 3, 2, 5]                       # repeated ids get blocks of their own
    _, e = eng.count_graphs(gids)
    values = np.random.default_rng(n).random(int(e.sum())).astype(np.float32)
    want = _host_densify(eng, gids, values)
    assert np.array_equal(eng.densify_graphs_host(gids, values), want)
    got = eng.densify_graphs_device(gids, torch.from_numpy(values).cuda())
    assert got.dtype == torch.float64 and np.array_equal(got.cpu().numpy(), want)
    out = torch.full((len(gids), n, n), 7.0, dtype=torch.float64, device="cuda")   # zero fill of a dirty buffer
    eng.densify_graphs_device(gids, torch.from_numpy(values).cuda(), out=out)
    assert np.array_equal(out.cpu().numpy(), want)
    assert eng.densify_graphs_host([], np.zeros(0, np.float32)).shape == (0, n, n)
    assert eng.densify_graphs_device([], torch.zeros(0, device="cuda")).shape == (0, n, n)
    for bad in ([12], [0, -1]):
        with pytest.raises(_abi.GnnxError) as e:
            eng.densify_graphs_host(bad, values)
        assert e.value.status == GX_ERR_INVALID
        with pytest.raises(_abi.GnnxError) as e:
            eng.count_graphs(bad)
        assert e.value.status == GX_ERR_INVALID
    eng.close()


def test_densify_and_count_need_a_batch():
    eng = gnnx.Engine(0)
    for call in (lambda: eng.count_graphs([0]), lambda: eng.densify_graphs_host([0], np.zeros(1, np.float32))):
        eng.batch_n = 1
        with pytest.raises(_abi.GnnxError) as e:
            call()
        assert e.value.status == GX_ERR_INVALID
    eng.close()


def test_densify_graphs_beyond_2_31_elements():
    """129 graphs of 4096 padded rows: 2.16e9 doubles (17 GB), past 32-bit indexing.  The last graph and zero elsewhere are checked."""
    G, n = 129, 4096
    rng = np.random.default_rng(1)
    eng = gnnx.Engine(0)
    # every graph a path over its first k rows (the last one over all 4096), uploaded as block CSR
    ks = rng.integers(2, 60, G)
    ks[-1] = n
    rowptr = np.zeros(G * n + 1, np.int64)
    cols = []
    for g, k in enumerate(ks):
        deg = np.zeros(n, np.int64)
        deg[:k] = 2
        deg[0] = deg[k - 1] = 1
        rowptr[g * n + 1:(g + 1) * n + 1] = deg
        for i in range(k):
            cols.append([j for j in (i - 1, i + 1) if 0 <= j < k])
    rowptr = np.cumsum(rowptr).astype(np.int32)
    col = np.array([j for c in cols for j in c], np.int32)
    feat, label = np.zeros(G * n, np.float32), np.zeros(G, np.int32)
    _abi.check(eng._lib.gx_set_graph_batch_csr(eng._h, G, n, rowptr.ctypes.data, col.ctypes.data, feat.ctypes.data, 1, label.ctypes.data))
    eng.batch_n = n
    eng.batch_rowptr, eng.batch_col = rowptr, col
    gids = list(range(G))
    n_c, e_c = eng.count_graphs(gids)
    assert np.array_equal(n_c, ks) and np.array_equal(e_c, 2 * (ks - 1))
    values = torch.from_numpy(rng.random(int(e_c.sum())).astype(np.float32)).cuda()
    out = eng.densify_graphs_device(gids, values)
    assert out.numel() > 2 ** 31
    last = out[-1].cpu().numpy()
    assert np.array_equal(last, _host_densify(eng, [G - 1], values[-int(e_c[-1]):].cpu().numpy())[0])
    head = values[:-int(e_c[-1])]                   # values in (0, 1): every other slot lands once, zeros around it
    assert int(torch.count_nonzero(out[:-1])) == head.numel()
    assert abs(float(out[:-1].sum()) - float(head.double().sum())) <= 1e-9 * head.numel()
    del out
    eng.close()


def test_count_graphs_matches_the_plan(gg):
    rng = np.random.default_rng(4)
    sizes = [6, 15, 30, 3]
    adj = _batch([_ba(s) for s in sizes] + [np.zeros((5, 5), np.uint8)], 32)
    eng = gnnx.Engine(0)
    eng.set_model({k: gg[k] for k in util.WKEYS})
    eng.set_graph_batch(adj, rng.normal(size=(len(adj), 32, 14)).astype(np.float32), np.zeros(len(adj), np.int32))
    gids = [2, 0, 4, 1, 3, 2]
    n_c, e_c = eng.count_graphs(gids)
    assert np.array_equal(e_c, np.diff(eng.plan_graphs(gids)))
    assert np.array_equal(n_c, [int((adj[g].sum(1) > 0).sum()) for g in gids])
    assert e_c[2] == 0 and n_c[2] == 0
    assert [len(x) for x in eng.count_graphs([])] == [0, 0]
    eng.close()
