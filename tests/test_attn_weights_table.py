"""Per-sample attn_weights on the host, without a device: the table the attention kernels read, the longest vector each
sample takes (the smallest key count it sees in an AttnBlock), and the ValueErrors raised before anything is enqueued."""
import pytest
import torch

from helpers import load_golden
from paella_b200 import ops


def test_table_rows_lengths_and_padding():
    a, b = torch.tensor([0.4, 1.2, 3.0]), torch.tensor([2.0], dtype=torch.float64)
    table, lens = ops.attn_weights_table([a, None, b, torch.zeros(0)], 4, [10] * 4)
    assert table.dtype == torch.float32 and lens.dtype == torch.int32
    assert table.shape == (4, 3) and lens.tolist() == [3, 0, 1, 0]
    assert torch.equal(table[0], a) and table[2].tolist() == [2.0, 0.0, 0.0]
    assert not table[1].any() and not table[3].any()
    table, lens = ops.attn_weights_table((None, None), 2, [5, 5])       # every row unweighted: one zero column
    assert table.shape == (2, 1) and lens.tolist() == [0, 0]


def test_table_bytes_survive_the_packed_copy_layout():
    """attn_weights_to_device sends the float table and the lengths as one int32 buffer; the views must round-trip."""
    table, lens = ops.attn_weights_table([torch.tensor([0.1, -2.5]), torch.tensor([7.0])], 2, [4, 4])
    flat = torch.cat([table.view(torch.int32).view(-1), lens])
    assert torch.equal(flat[:table.numel()].view(torch.float32).view(table.shape), table)
    assert torch.equal(flat[table.numel():], lens)


@pytest.mark.parametrize("bad", [
    [torch.ones(3)],                                      # too few entries
    [torch.ones(3)] * 3,                                  # too many
    [torch.ones(3), torch.ones(2, 2)],                    # not 1-D
    [torch.ones(3), torch.ones((), dtype=torch.float32)],  # 0-D
    [torch.ones(3), torch.ones(3, dtype=torch.int64)],    # not floating point
    [torch.ones(3), torch.tensor([1.0, float("nan")])],
    [torch.ones(3), torch.tensor([float("inf")])],
    [torch.ones(3), torch.ones(6)],                       # longer than the smallest key count (5)
    [torch.ones(3), [1.0, 2.0]],                          # not a tensor
])
def test_bad_tables_raise_value_error(bad):
    with pytest.raises(ValueError):
        ops.attn_weights_table(bad, 2, [5, 5])


def test_max_attn_weights_is_the_smallest_key_count():
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    with torch.device("meta"):
        m = Paella(**cfg)
    ps = cfg["patch_size"]
    levels = [i for i, (kinds, n) in enumerate(zip(cfg["level_config"], cfg["blocks"])) if "A" in kinds and n > 0]
    assert levels, "the tiny model has AttnBlocks"
    for H, W, S in [(8, 8, 7), (16, 8, 12), (32, 32, 0)]:
        want = min(((H // ps) >> i) * ((W // ps) >> i) * int(cfg.get("self_attn", True)) + S for i in levels)
        assert m.max_attn_weights((H, W), S) == want
    with torch.device("meta"):
        d = Paella()
    assert d.max_attn_weights((32, 32), 77) == 4 * 4 + 77       # the default model's deepest level is 4x4 at 32x32 tokens
    with torch.device("meta"):
        no_self = Paella(**dict(cfg, self_attn=False))
    assert no_self.max_attn_weights((8, 8), 9) == 9             # cross-attention only: the conditioning rows
