"""CPU tests of the plan's symbolic-tensor bookkeeping (no kernel runs)."""
import torch

from centerpose_b200.plan import PlanBuilder


def _conv(pb, srcs, co):
    return pb.conv(srcs, torch.zeros(co, sum(s.C for s in srcs), 1, 1), torch.zeros(co))


def test_channel_slice_keeps_parent_buffer_live():
    """A channel slice is read from its parent's buffer at the slice's channel offset, with the parent's pitch, and it
    keeps the parent live: after the parent's last direct reader, the parent's buffer goes to no other op until the
    slice has been read, and is reused after that."""
    pb = PlanBuilder(1, 8, 8, "fp32", torch.device("cpu"))
    x = pb.external(torch.zeros(1, 8, 8, 16))
    p = _conv(pb, [x], 64)                      # op 0
    s = pb.channel_slice(p, 48, 16)
    q = _conv(pb, [p], 64)                      # op 1: the parent's last direct reader
    _conv(pb, [q], 64)                          # op 2: would take the parent's buffer if the slice did not keep it live
    t = _conv(pb, [s], 64)                      # op 3: reads the slice
    pb.keep_result(_conv(pb, [t], 64))          # op 4: takes the parent's buffer
    plan = pb.build()
    assert plan.n == 5 and (p.pitch, s.pitch, x.pitch) == (64, 64, 16)
    assert s.buf is p.buf
    base = p.buf.data_ptr()
    assert (plan.ops[1].src[0], plan.ops[1].src_pitch[0]) == (base, 0)
    assert (plan.ops[3].src[0], plan.ops[3].src_pitch[0]) == (base + 48 * 4, 64)
    assert [plan.ops[i].dst == base for i in range(5)] == [True, False, False, False, True]
