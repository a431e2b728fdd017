"""SamplingEngine admission grouping on the host (no GPU): which conditioning slots one prepare_cond call projects together."""
import torch

from paella_b200.engine import admission_runs, cond_layout


def _inputs(L, clip=True, n_img=0, as_list=False):
    d = {"byt5": torch.zeros(1, L, 8)}
    if clip:
        d["clip"] = torch.zeros(1, 4)
    if n_img:
        imgs = [torch.zeros(1, 4) for _ in range(n_img)]
        d["clip_image"] = imgs if (as_list or n_img > 1) else imgs[0]
    return d


def test_cond_layout():
    assert cond_layout(_inputs(128)) == (128, True, 0)
    assert cond_layout(_inputs(77, clip=False)) == (77, False, 0)
    assert cond_layout(_inputs(10, n_img=1)) == (10, True, 1)
    assert cond_layout(_inputs(10, n_img=1, as_list=True)) == (10, True, 1)
    assert cond_layout(_inputs(10, clip=False, n_img=3)) == (10, False, 3)


def _runs(writes):
    return [[writes[i][0] for i in run] for run in admission_runs(writes)]


def test_one_layout_contiguous_slots_is_one_run():
    a = cond_layout(_inputs(128))
    assert _runs([(s, a) for s in range(5)]) == [[0, 1, 2, 3, 4]]
    assert _runs([]) == []


def test_runs_break_at_layout_changes_and_slot_gaps():
    a, b = cond_layout(_inputs(128)), cond_layout(_inputs(64, clip=False))
    # mixed layouts on contiguous slots
    assert _runs([(0, a), (1, a), (2, b), (3, a)]) == [[0, 1], [2], [3]]
    # non-contiguous free slots (a retired request freed 1 and 4): same layout, separate runs
    assert _runs([(0, a), (2, a), (3, a), (5, a)]) == [[0], [2, 3], [5]]
    # the same layout but a different number of clip images is another layout
    assert _runs([(0, cond_layout(_inputs(8, n_img=1))), (1, cond_layout(_inputs(8, n_img=2)))]) == [[0], [1]]


def test_runs_are_in_slot_order_and_cover_every_write_once():
    a, b = cond_layout(_inputs(128)), cond_layout(_inputs(64))
    writes = [(7, a), (3, b), (4, b), (6, a), (2, b), (9, a)]
    runs = admission_runs(writes)
    assert sorted(i for r in runs for i in r) == list(range(len(writes)))
    assert [[writes[i][0] for i in r] for r in runs] == [[2, 3, 4], [6, 7], [9]]


def test_own_unconditional_slots_group_like_the_conditional_ones():
    # the engine writes request slot s and its own unconditional slot max_batch + s; requests that use the engine-wide
    # shared unconditional slot contribute no second write
    max_batch = 8
    cond, unc, unc2 = cond_layout(_inputs(128)), cond_layout(_inputs(128, clip=False)), cond_layout(_inputs(16, clip=False))
    reqs = [(0, unc), (1, unc), (2, None), (3, unc), (4, unc)]          # (slot, layout of its own negative prompt or None)
    writes = [(s, cond) for s, _ in reqs] + [(max_batch + s, u) for s, u in reqs if u is not None]
    assert _runs(writes) == [[0, 1, 2, 3, 4], [8, 9], [11, 12]]
    # a request whose negative prompt has another layout splits the unconditional run
    reqs[1] = (1, unc2)
    writes = [(s, cond) for s, _ in reqs] + [(max_batch + s, u) for s, u in reqs if u is not None]
    assert _runs(writes) == [[0, 1, 2, 3, 4], [8], [9], [11, 12]]
