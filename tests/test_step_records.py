"""The records of one bilevel step, merged and filed on the host (no device): fused.merge keeps a video's last evaluation when a
later loop iteration leaves it out, and multivideo.slot_records fills idle slots with NaN and keeps their last_upper_loss."""
import math

import torch

from dynaboa_b200.fused import Frame, merge, pick
from dynaboa_b200.multivideo import slot_records

NAN = float('nan')


def same(a, b):
    return all((math.isnan(x) and math.isnan(y)) or x == y for x, y in zip(a.tolist(), b.tolist()))


def test_pick():
    a, b = torch.tensor([1., 2., 3., 4.]), torch.tensor([5., 6., 7., 8.])
    assert pick(0b1111, 4, a, b) is a                               # every video: the tensor itself, nothing launched
    assert same(pick(0b0101, 4, a, b), torch.tensor([1., 6., 3., 8.]))
    assert same(pick(0b0101, 4, a), torch.tensor([1., NAN, 3., NAN]))


def test_a_video_outside_a_loop_iteration_keeps_its_last_value():
    upper = {'ul/s2dloss': torch.tensor([1., 2., 3., 4.]), 'ul/motion_loss': torch.tensor([.1, .2, .3, .4])}
    loop = {'ul/s2dloss': torch.tensor([10., 20., 30., 40.]), 'ul/labled_loss': torch.tensor([5., 6., 7., 8.])}
    out = merge(upper, loop, 0b0110, 4)                             # videos 1 and 2 ran the iteration
    assert list(out) == ['ul/s2dloss', 'ul/motion_loss', 'ul/labled_loss']
    assert same(out['ul/s2dloss'], torch.tensor([1., 20., 30., 4.]))
    assert out['ul/motion_loss'] is upper['ul/motion_loss']         # not evaluated again: kept for every video
    assert out['ul/labled_loss'] is loop['ul/labled_loss']          # first evaluated here
    assert upper['ul/s2dloss'].tolist() == [1., 2., 3., 4.]         # the records merged are not modified
    full = merge(upper, loop, 0b1111, 4)
    assert full['ul/s2dloss'] is loop['ul/s2dloss']


def test_idle_slots_get_nan_and_keep_their_upper_loss():
    f = Frame(0b1010)                                               # slots 1 and 3 advanced this frame
    f.fit = {'ll/s2dloss': torch.tensor([9., 1., 9., 3.]), 'feat_sim/cos_sim': torch.tensor([9., .5, 9., .7])}
    f.lower = [torch.tensor([9., 1., 9., 3.]), torch.tensor([9., 2., 9., 4.])]
    f.upper_loss = torch.tensor([9., 10., 9., 30.])
    prev = torch.tensor([100., 200., 300., 400.])
    fit, lower, loss = slot_records(f, 4, prev)
    assert same(fit['ll/s2dloss'], torch.tensor([NAN, 1., NAN, 3.]))
    assert same(fit['feat_sim/cos_sim'], torch.tensor([NAN, .5, NAN, .7]))
    assert [x.tolist()[1::2] for x in lower] == [[1., 3.], [2., 4.]] and all(math.isnan(v) for x in lower for v in x.tolist()[::2])
    assert same(loss, torch.tensor([100., 10., 300., 30.]))
    assert prev.tolist() == [100., 200., 300., 400.]


def test_a_full_frame_is_filed_as_it_is():
    f = Frame(0b11)
    f.fit, f.lower, f.upper_loss = {'ul/s2dloss': torch.tensor([1., 2.])}, [], torch.tensor([3., 4.])
    fit, lower, loss = slot_records(f, 2, torch.tensor([0., 0.]))
    assert fit['ul/s2dloss'] is f.fit['ul/s2dloss'] and lower == [] and loss is f.upper_loss
