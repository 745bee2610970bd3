"""Full parameter sharding under amp_fp8, host side: the per-rank pieces of the block weight matrices that each owner quantises into
its E4M3 shard, and the memory table of the fp8 communicator."""
import pytest

MC = {"name": "mpt_causal_lm", "d_model": 128, "n_heads": 4, "n_layers": 12, "expansion_ratio": 4, "max_seq_len": 64, "vocab_size": 512}


@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_weight_pieces_tile_every_block_matrix_once(n):
    from photon_b200.models.engine import B200Engine
    from photon_b200.parallel.zero3 import BLOCK_MATRICES, UnitPlan
    from photon_b200.utils.flat import layout_for_model_cfg

    lay = layout_for_model_cfg(MC)
    pl = UnitPlan(lay, 12, n)
    names = pl.weight_names
    assert len(names) == 4 * 12 and len(set(names)) == len(names)
    # slot j = block j // 4, matrix j % 4: the order of the engine's weight roles (block by block, wqkv / wo / wup / wdown)
    keys = dict(zip(BLOCK_MATRICES, B200Engine._W_ROLES))
    assert list(keys.values()) == list(B200Engine._W_ROLES)
    for j, name in enumerate(names):
        assert name == f"transformer.blocks.{j // 4}.{BLOCK_MATRICES[j % 4]}" and len(lay.shapes[lay.index(name)]) == 2
    # every 2-D tensor of a block unit is one of them (nothing else of a block needs a bf16 gather under fp8)
    assert {nm for nm, shp in zip(lay.names, lay.shapes) if ".blocks." in nm and len(shp) == 2} == set(names)
    covered = {name: [] for name in names}
    for r in range(n):
        pieces = pl.weight_pieces(r)
        ends = sorted((o, o + k) for o, k, _ in pieces)
        assert all(a[1] <= b[0] for a, b in zip(ends, ends[1:])), "pieces of one shard overlap"
        assert all(0 <= o and o + k <= pl.shard_len for o, k, _ in pieces)
        for o, k, j in pieces:
            assert o % 8 == 0 and k % 8 == 0 and k > 0
            u, rel, ne = pl.rel(names[j])
            un = pl.units[u]
            # the piece lies inside rank r's slice of the matrix's unit, at the flat position it stands for
            assert un.off <= o and o + k <= un.off + un.per
            flat_lo = un.lo + r * un.per + (o - un.off)
            assert lay.offsets[lay.index(names[j])] <= flat_lo and flat_lo + k <= lay.offsets[lay.index(names[j])] + ne
            covered[names[j]].append((flat_lo, flat_lo + k))
    for name, spans in covered.items():
        spans.sort()
        i = lay.index(name)
        assert spans[0][0] == lay.offsets[i] and spans[-1][1] == lay.offsets[i] + lay.numels[i], name
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:])), name     # exactly once, no gaps
        assert len(spans) <= n                                                # at most one piece per rank


def test_pieces_gathered_bytes_equal_the_flat_layout():
    """What the E4M3 gather assembles: rank r's shard bytes of unit u land at r * per inside the unit buffer, so every piece is at
    its flat position relative to the unit (the views the engine's fp8 GEMMs read)."""
    import torch

    from photon_b200.parallel.zero3 import UnitPlan
    from photon_b200.utils.flat import layout_for_model_cfg

    lay = layout_for_model_cfg(MC)
    for n in (2, 3):
        pl = UnitPlan(lay, 12, n)
        full = torch.arange(lay.total, dtype=torch.float64)
        shards = [pl.full_to_shard(full, r, torch.empty(pl.shard_len, dtype=torch.float64)) for r in range(n)]
        for r in range(n):
            for o, k, j in pl.weight_pieces(r):
                u, rel, _ = pl.rel(pl.weight_names[j])
                un = pl.units[u]
                unit_buf_pos = r * un.per + (o - un.off)
                assert torch.equal(shards[r][o: o + k], full[un.lo + unit_buf_pos: un.lo + unit_buf_pos + k])


@pytest.mark.parametrize("n", [1, 2, 8])
def test_fp8_memory_table(n):
    from photon_b200.parallel.zero3 import UnitPlan
    from photon_b200.utils.flat import layout_for_model_cfg

    pl = UnitPlan(layout_for_model_cfg(MC), 12, n)
    plain, fp8 = pl.bytes_per_rank(), pl.bytes_per_rank(fp8=True)
    assert pl.bytes_per_rank() == plain and set(plain) < set(fp8)      # the default table is unchanged
    assert fp8["unit_weight_buffers_bf16"] == 2 * pl.rest_span         # the embeddings only: no bf16 block buffers
    assert fp8["unit_weight_buffers_e4m3"] == 2 * pl.max_block_span    # two rotating E4M3 units, one byte per element
    assert fp8["e4m3_shard"] == pl.shard_len
    assert fp8["amax_fp32"] == 4 * (n + 1) * 4 * 12                    # world rows of the amax plane + this rank's partials
    assert all(fp8[k] == plain[k] for k in plain if k != "unit_weight_buffers_bf16")
