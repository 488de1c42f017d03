"""The write-footprint harness of tests/footprint.py: its table covers every public ops function, and check_footprint
catches each kind of violation it claims to. The violations are planted in torch-only stand-ins registered as temporary
ops, so no kernel is involved; the same cases run on the GPU in tests/test_write_footprint_gpu.py."""
import pytest
import torch

import footprint as F
from fsb200 import ops

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


def test_every_ops_function_has_a_write_entry():
    missing = F.missing_entries()
    assert not missing, f"ops.{missing[0]} has no write-footprint entry (WRITES in tests/footprint.py)"


def test_a_deleted_entry_is_named(monkeypatch):
    monkeypatch.delitem(F.WRITES, "kv_append")
    assert F.missing_entries() == ["kv_append"]


# ------------------------------------------------------------------------------------------------- planted violations
def _exact(x, out):
    out.copy_(x)
    return out


def _past_end(x, out):
    out.copy_(x)
    torch.as_strided(out, (out.numel() + 1,), (1,), out.storage_offset())[-1] = 1.0   # one element past the view
    return out


def _one_short(x, out):
    out[:-1].copy_(x[:-1])
    return out


def _touches_input(x, out):
    out.copy_(x)
    x[3] += 1.0
    return out


def _past_workspace(x, out):
    ws = ops.workspace(64, x.device, "standin")
    torch.as_strided(ws, (68,), (1,), ws.storage_offset())[64:].fill_(0)                # one float past the workspace
    out.copy_(x)
    return out


def _fresh_short(x, out):
    y = ops.torch.empty_like(x)
    y[1:].copy_(x[1:])
    out.copy_(x)
    return y


def _register(monkeypatch, fn):
    monkeypatch.setattr(ops, "standin", fn, raising=False)
    monkeypatch.setitem(F.WRITES, "standin", lambda a: [F.Write("out", a["out"], F.OVERWRITE)])


def _arena(device):
    """x and out inside one sentinel-filled arena: out = arena[32:48], x = arena[64:80]."""
    arena = torch.full((128,), -3.0, device=device)
    arena[64:80] = torch.arange(16, dtype=torch.float32, device=device)
    return arena, arena[64:80], arena[32:48]


@pytest.mark.parametrize("device", DEVICES)
def test_a_call_within_its_footprint_passes(device, monkeypatch):
    _register(monkeypatch, _exact)
    arena, x, out = _arena(device)
    before = arena.clone()
    F.check_footprint("standin", ops.standin, (x, out), {}, F.Stats())
    assert torch.equal(out, x) and torch.equal(arena[:32], before[:32]) and torch.equal(arena[48:], before[48:])


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("fn, message", [
    (_past_end, r"ops\.standin: \d bytes changed outside the declared writes in the storage of argument\(s\) "
                r"\['x', 'out'\], outside every argument view; first at storage byte offset 19[2-5]"),
    (_one_short, r"ops\.standin: 1/16 elements of the overwrite argument 'out' were never written"),
    (_touches_input, r"ops\.standin: \d bytes changed outside the declared writes in argument 'x'; first at storage "
                     r"byte offset 2(6[89]|7[01])"),
    (_past_workspace, r"ops\.standin: workspace 'standin' \(64 bytes\): 4 guard bytes after it changed, first at byte 64"),
    (_fresh_short, r"ops\.standin: 1/16 elements of the tensor it allocated \(#0, \(16,\) torch\.float32\) were never "
                   r"written"),
], ids=["past_end", "one_short", "touches_input", "past_workspace", "fresh_short"])
def test_a_planted_violation_fails_by_op_and_argument(fn, message, device, monkeypatch):
    _register(monkeypatch, fn)
    arena, x, out = _arena(device)
    with pytest.raises(AssertionError, match=message):
        F.check_footprint("standin", ops.standin, (x, out), {}, F.Stats())


def test_an_op_without_entry_fails_by_name():
    with pytest.raises(AssertionError, match=r"ops\.add has no write-footprint entry"):
        saved = F.WRITES.pop("add")
        try:
            F.check_footprint("add", ops.add, (torch.ones(8), torch.ones(8)), {}, F.Stats())
        finally:
            F.WRITES["add"] = saved


def test_an_overwrite_that_aliases_an_input_is_not_poisoned(monkeypatch):
    """out= x: fsb_add / fsb_dropout allow it, so the view is an update and x is not destroyed before the call."""
    _register(monkeypatch, lambda x, out: out.mul_(2.0))
    x = torch.arange(16, dtype=torch.float32)
    F.check_footprint("standin", ops.standin, (x, x), {}, F.Stats())
    assert torch.equal(x, 2.0 * torch.arange(16, dtype=torch.float32))


def test_poison_never_equals_a_code_the_quantisers_write():
    """int8 codes are clamped to [-127, 127]; int4 nibbles are q + 8 in 1 .. 15; FP8 0x7f is NaN in e4m3 and e5m2."""
    q8 = torch.arange(-127, 128, dtype=torch.int8)
    assert not F.poisoned(q8).any()
    nib = torch.arange(1, 16, dtype=torch.uint8)
    assert not F.poisoned((nib[:, None] | (nib[None, :] << 4)).reshape(-1)).any()
    for dt in (torch.float8_e4m3fn, torch.float8_e5m2):
        t = torch.empty(4, dtype=dt)
        F.poison(t)
        assert torch.isnan(t.float()).all()
