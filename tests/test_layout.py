"""Shard arithmetic property tests: pad / chunk / un-pad round-trips for arbitrary shapes and world sizes."""
import torch
from hypothesis import given, settings, strategies as st

from vit_10b_fsdp_example_b200.parallel.layout import ALIGN, UnitLayout

shapes = st.lists(st.lists(st.integers(1, 37), min_size=1, max_size=3), min_size=1, max_size=6)


@settings(max_examples=60, deadline=None)
@given(shapes=shapes, world=st.integers(1, 8), flatten=st.booleans())
def test_round_trip(shapes, world, flatten):
    specs = [(f"p{i}", tuple(s)) for i, s in enumerate(shapes)]
    lay = UnitLayout.build("u", specs, world, flatten)
    assert lay.full_numel % ALIGN == 0 and lay.shard_numel % ALIGN == 0
    assert lay.shard_numel * world == lay.full_numel
    full = torch.zeros(lay.full_numel)
    for i, p in enumerate(lay.params):
        assert p.full_offset % ALIGN == 0
        full[p.full_offset: p.full_offset + p.numel] = torch.arange(p.numel, dtype=torch.float32) + 1000 * (i + 1)
    shards = [lay.shard_from_full(full, r, torch.zeros(lay.shard_numel)) for r in range(world)]
    back = lay.full_from_shards(shards, torch.zeros(lay.full_numel))
    assert torch.equal(back, full)
    # gather segments cover every rank's shard exactly once and land in disjoint destinations
    covered = torch.zeros(lay.full_numel, dtype=torch.int32)
    for (r, soff, doff, n) in lay.gather_segments():
        covered[doff: doff + n] += 1
        assert torch.equal(full[doff: doff + n], shards[r][soff: soff + n])
    assert int(covered.max()) == 1 and int(covered.sum()) == lay.full_numel
    # views have the declared shapes; metadata round-trips
    views = lay.param_views(full)
    for p in lay.params:
        assert tuple(views[p.name].shape) == p.shape
    lay2 = UnitLayout.from_metadata(lay.metadata())
    assert lay2.metadata() == lay.metadata()


def test_vit10b_block_layout_numbers():
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.models import vit

    cfg = ViTConfig()
    assert cfg.block_numel() == 314_639_360
    assert cfg.total_numel() == 10_077_917_160        # "10 billion parameters"
    lay = UnitLayout.build("blocks.0", vit.block_param_specs(cfg), 8, False)
    assert lay.payload_numel() == cfg.block_numel()
    assert lay.shard_numel * 8 == lay.full_numel
    assert lay.full_numel - cfg.block_numel() < 12 * 8 * ALIGN


def test_split_fp32_is_exact_including_ties():
    """(bf16 hi, int16 lo) must reproduce every fp32 bit pattern, also exact rounding ties and negatives."""
    from vit_10b_fsdp_example_b200.ops import torch_ops

    bits = torch.tensor([0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F807FFF, 0x3F808001, 0x00000000,
                         0x80000000, 0x3F7FFFFF, 0x7F7FFFFF], dtype=torch.int64).to(torch.int32)
    w = torch.cat([bits.view(torch.float32), torch.randn(4096)])
    hi = torch.empty(w.numel(), dtype=torch.bfloat16)
    lo = torch.empty(w.numel(), dtype=torch.int16)
    torch_ops.split_fp32(w, hi, lo)
    back = torch.empty_like(w)
    torch_ops.merge_fp32(hi, lo, back)
    assert torch.equal(back.view(torch.int32), w.view(torch.int32))
