"""CPU: the host side of graph-mode sharding (gnnx.dist.explain_graphs_sharded) without a GPU: the torch-compatible M0 draw of one rank's
graphs against a single process's draw, and the shard layout from per-graph costs."""
import math
import types

import numpy as np
import pytest
import torch

import conftest  # noqa: F401  (sys.path)
from gnnx import dist as gdist
from gnnx.explain import Explainer


def _padded_graphs(rng, n, G):
    """(rows, cols) in slot order of G random symmetric graphs padded to n rows; graph 2 has no edge."""
    out = []
    for g in range(G):
        k = 0 if g == 2 else int(rng.integers(2, n))
        A = np.zeros((n, n), np.uint8)
        a, b = rng.integers(0, k, 3 * k), rng.integers(0, k, 3 * k)
        ok = a != b
        A[a[ok], b[ok]] = 1
        A[b[ok], a[ok]] = 1
        r, c = np.nonzero(A)
        out.append((r.astype(np.int64), c.astype(np.int64)))
    return out


def _single_process(n, rcs):
    """Explainer._explain_graph_batch's draw: FloatTensor(n, n).normal_(1, std) per graph in list order, n = the padded size."""
    std = torch.nn.init.calculate_gain("relu") * math.sqrt(2.0 / (n + n))
    return [torch.FloatTensor(n, n).normal_(1.0, std).numpy()[r, c] for r, c in rcs]


@pytest.mark.parametrize("n", [7, 33])
def test_draw_graph_m0_subset_matches_one_process(n):
    rng = np.random.default_rng(n)
    G = 11
    rcs = _padded_graphs(rng, n, G)
    sizes = np.array([len(r) for r, _ in rcs])
    torch.manual_seed(123)
    want = _single_process(n, rcs)
    state_after = torch.get_rng_state()
    for world in (1, 2, 3, 4):
        shards = gdist.shard_layout(sizes, world)[0]
        for rank in range(world):
            pos = shards[rank]
            torch.manual_seed(123)
            got = Explainer._draw_graph_m0_subset(n, G, pos, [rcs[p] for p in pos])
            assert torch.equal(torch.get_rng_state(), state_after), (world, rank)
            assert got.dtype == np.float32
            expect = np.concatenate([want[p] for p in pos]) if len(pos) else np.zeros(0, np.float32)
            assert np.array_equal(got, expect), (world, rank)


def test_draw_graph_m0_subset_owning_nothing_still_walks_the_list():
    torch.manual_seed(5)
    _single_process(9, [(np.zeros(0, np.int64), np.zeros(0, np.int64))] * 4)
    state_after = torch.get_rng_state()
    torch.manual_seed(5)
    got = Explainer._draw_graph_m0_subset(9, 4, np.zeros(0, np.int64), [])
    assert got.size == 0 and torch.equal(torch.get_rng_state(), state_after)


def test_shard_layout_from_graph_costs():
    rng = np.random.default_rng(2)
    rcs = _padded_graphs(rng, 40, 57)
    e_d = np.array([len(r) for r, _ in rcs], np.int64)       # gx_count_graphs' e_out: the default cost and the payload of every graph
    for world in (1, 2, 4, 8):
        shards, slot, src_off, offsets = gdist.shard_layout(e_d, world)
        assert np.array_equal(np.sort(np.concatenate(shards)), np.arange(len(e_d)))
        assert offsets[0] == 0 and np.array_equal(np.diff(offsets), e_d)
        payload = [int(e_d[s].sum()) for s in shards]
        assert slot == max(max(payload), 1) and max(payload) - min(payload) <= e_d.max()
        for r, s in enumerate(shards):
            assert np.array_equal(src_off[s], r * slot + np.concatenate([[0], np.cumsum(e_d[s])[:-1]]))
        # explicit costs move graphs between ranks, the payload sizes stay the edges
        costs = e_d + 4 * np.arange(len(e_d))
        shards_c, slot_c, _, offsets_c = gdist.shard_layout(e_d, world, costs)
        assert np.array_equal(offsets_c, offsets) and slot_c == max(max(int(e_d[s].sum()) for s in shards_c), 1)
        assert np.array_equal(shards_c[0], np.sort(np.argsort(-costs, kind="stable")[0::world]))


def test_sharded_graph_mode_needs_graph_mode():
    with pytest.raises(ValueError, match="graph_mode=True"):
        gdist.explain_graphs_sharded(types.SimpleNamespace(graph_mode=False), [0, 1])
