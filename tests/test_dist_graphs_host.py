"""CPU: the host side of sharding (gnnx.dist) without a GPU: the torch-compatible M0 walk (gnnx.explain.torch_m0_walk) kept at one rank's
entries, graph mode (also through Explainer._draw_graph_m0_subset) and node mode, against a single process's draw, and the shard layout from
per-graph costs."""
import types

import numpy as np
import pytest
import torch

import conftest  # noqa: F401  (sys.path)
from gnnx import dist as gdist
from gnnx.explain import Explainer, torch_m0_walk
import gnnx_oracle as O


def _edge_lists(rng, sizes):
    """(rows, cols) in slot order of random symmetric graphs of sizes[p] rows each; entry 2 has no edge."""
    out = []
    for g, n in enumerate(sizes):
        k = 0 if g == 2 else int(rng.integers(2, n))
        A = np.zeros((n, n), np.uint8)
        a, b = rng.integers(0, k, 3 * k), rng.integers(0, k, 3 * k)
        ok = a != b
        A[a[ok], b[ok]] = 1
        A[b[ok], a[ok]] = 1
        r, c = np.nonzero(A)
        out.append((r.astype(np.int64), c.astype(np.int64)))
    return out


def _single_process(sizes, rcs):
    """The reference's draw of every list entry in list order (ExplainModule.construct_edge_mask), at the entry's slots."""
    return [O.draw_m0(n)[r, c] for n, (r, c) in zip(sizes, rcs)]


# graph mode: every graph padded to one size; node mode: a k-hop size per list entry
@pytest.mark.parametrize("sizes", [[7] * 11, [33] * 11, [5, 31, 3, 18, 40, 9, 3, 27, 12, 6, 20], [4, 64, 17, 3, 45, 8, 23, 3]],
                         ids=["graphs7", "graphs33", "nodes11", "nodes8"])
def test_m0_walk_matches_one_process(sizes):
    rng = np.random.default_rng(sizes[0])
    rcs = _edge_lists(rng, sizes)
    e_d = np.array([len(r) for r, _ in rcs])
    torch.manual_seed(123)
    want = _single_process(sizes, rcs)
    state_after = torch.get_rng_state()
    for world in (1, 2, 3, 4):
        shards = gdist.shard_layout(e_d, world)[0]
        for rank in range(world):
            pos = shards[rank]
            torch.manual_seed(123)
            mine = set(pos.tolist())
            kept = [M[rcs[p]] for p, M in enumerate(torch_m0_walk(sizes)) if p in mine]
            assert torch.equal(torch.get_rng_state(), state_after), (world, rank)
            got = np.concatenate(kept) if kept else np.zeros(0, np.float32)
            assert got.dtype == np.float32
            expect = np.concatenate([want[p] for p in pos]) if len(pos) else np.zeros(0, np.float32)
            assert np.array_equal(got, expect), (world, rank)
            if len(set(sizes)) == 1:       # graph mode: what explain_graphs_sharded draws on this rank
                torch.manual_seed(123)
                got = Explainer._draw_graph_m0_subset(sizes[0], len(sizes), pos, [rcs[p] for p in pos])
                assert torch.equal(torch.get_rng_state(), state_after), (world, rank)
                assert got.dtype == np.float32
                assert np.array_equal(got, expect), (world, rank)


def test_draw_graph_m0_subset_owning_nothing_still_walks_the_list():
    torch.manual_seed(5)
    _single_process([9] * 4, [(np.zeros(0, np.int64), np.zeros(0, np.int64))] * 4)
    state_after = torch.get_rng_state()
    torch.manual_seed(5)
    got = Explainer._draw_graph_m0_subset(9, 4, np.zeros(0, np.int64), [])
    assert got.size == 0 and torch.equal(torch.get_rng_state(), state_after)


def test_shard_layout_from_graph_costs():
    rng = np.random.default_rng(2)
    rcs = _edge_lists(rng, [40] * 57)
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
