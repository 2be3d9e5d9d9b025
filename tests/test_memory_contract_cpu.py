"""The checks of tests/memory_contract.py on CPU tensors: each one fires on the fault it is there for and passes a clean
case, so that a GPU test built on them cannot pass vacuously."""
import pytest
import torch

import memory_contract as mc


def store(flat, i, v):
    """flat[i] = v, also for i just outside flat (into the guard that surrounds it)."""
    flat.as_strided((1,), (1,), flat.storage_offset() + i).fill_(v)


@pytest.mark.parametrize('offset', [0, 4, 12])
def test_a_clean_call_passes(offset):
    inp = torch.arange(35, dtype=torch.float32).view(5, 7)
    before = mc.snapshot([inp])
    g = mc.guarded((5, 7), offset, 'cpu')
    assert g.ptr() % 16 == offset % 16
    assert mc.n_unwritten(g.t) == 35 and g.untouched()
    g.t.copy_(2 * inp)
    mc.assert_written(g, 'out')
    assert mc.unchanged(before, [inp])
    assert not g.untouched()


@pytest.mark.parametrize('side', [-1, 35])
@pytest.mark.parametrize('fill', ['sentinel', 'zero'])
def test_a_one_element_overrun_on_either_side_breaks_a_guard(side, fill):
    g = mc.guarded((5, 7), 4, 'cpu')
    g.t.fill_(1.0)
    store(g.t.view(-1), side, 1.0)
    with pytest.raises(AssertionError, match='outside the buffer'):
        mc.assert_written(g, 'out')
    ws = mc.workspace(140, 4, fill, 'cpu')
    assert ws.guards_intact()
    ws.t.view(torch.float32).fill_(3.0)
    assert ws.guards_intact()
    store(ws.t.view(torch.float32), side, 3.0)
    assert not ws.guards_intact()


def test_a_workspace_guard_catches_one_byte_past_the_end():
    ws = mc.workspace(140, 0, 'zero', 'cpu')
    assert torch.count_nonzero(ws.t) == 0 and ws.guards_intact()
    ws.buf[ws.hi] = 0xA5 ^ 1
    assert not ws.guards_intact()


@pytest.mark.parametrize('where', [0, 17, 34])
def test_one_unwritten_element_is_found(where):
    g = mc.guarded((5, 7), 0, 'cpu')
    flat = g.t.view(-1)
    for i in range(35):
        if i != where:
            flat[i] = float(i)
    assert mc.n_unwritten(g.t) == 1
    with pytest.raises(AssertionError, match='1 of 35 elements never written'):
        mc.assert_written(g, 'out')


def test_a_computed_nan_counts_as_written_and_the_sentinel_is_a_nan():
    g = mc.guarded((4,), 0, 'cpu')
    assert torch.isnan(g.t).all()
    g.t.copy_(torch.tensor([0.0, -0.0, float('nan'), float('inf')]))
    mc.assert_written(g, 'out')


def test_one_mutated_input_is_found():
    inp = [torch.randn(3, 4), None, torch.randn(2)]
    before = mc.snapshot(inp)
    assert mc.unchanged(before, inp)
    inp[2][1] = inp[2][1].nextafter(torch.tensor(float('inf')))
    assert not mc.unchanged(before, inp)
    # a NaN input must keep its payload
    x = torch.tensor([1.0]).view(torch.int32).fill_(mc.SENTINEL).view(torch.float32)
    b = mc.snapshot([x])
    x.view(torch.int32).fill_(0x7FFFFFFF)
    assert torch.isnan(x).all() and not mc.unchanged(b, [x])


def test_same_bits_is_nan_aware_and_tells_signed_zeros_apart():
    a = torch.tensor([1.0, float('nan'), 0.0])
    b = a.clone()
    b.view(torch.int32)[1] = 0x7FFFFFFF                  # another NaN: the same
    assert mc.same_bits(a, b)
    b[2] = -0.0
    assert not mc.same_bits(a, b)
    b[2] = 0.0
    b[0] = 1.0000001
    assert not mc.same_bits(a, b)
    assert not mc.same_bits(a, a[:2])
    c = a.clone()
    c[1] = 5.0
    assert not mc.same_bits(a, c)
