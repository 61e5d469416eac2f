"""PreparedMixin (real3dportrait_b200/prepared.py) on small CPU modules: a value is built once and then served, its key separates modes, a
load_state_dict or a move / cast of the module or of an ancestor drops every entry, forget() drops one, and a watched module's in-place
edit or own load_state_dict triggers a rebuild that an unrelated module does not."""
import torch
import torch.nn as nn

from real3dportrait_b200.prepared import PreparedMixin


class _Counted(PreparedMixin, nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = nn.Linear(4, 4)
        self.builds = 0

    def build(self):
        self.builds += 1
        return self.lin.weight.detach() * 2


def _value(m, *key, watch=()):
    return m.prepared('w', m.build, *key, watch=watch)


def test_built_once_then_served():
    m = _Counted()
    v = _value(m)
    assert _value(m) is v and m.builds == 1
    assert m.cached('w') is v and m.cached('other') is None


def test_key_separates_modes():
    m = _Counted()
    a = _value(m, False)
    b = _value(m, True)
    assert b is not a and m.builds == 2
    assert m.cached('w', False) is None and m.cached('w', True) is b
    assert _value(m, True) is b and m.builds == 2


def test_load_state_dict_drops_entries_of_the_module_and_its_descendants():
    m = _Counted()
    parent = nn.Sequential(m)
    for loader, sd in ((m, m.state_dict()), (parent, parent.state_dict())):
        _value(m)
        m.store('clip', 'constants')
        n = m.builds
        loader.load_state_dict(sd)
        assert m.cached('w') is None and m.cached('clip') is None
        _value(m)
        assert m.builds == n + 1


def test_move_or_cast_drops_entries_of_the_module_and_its_descendants():
    m = _Counted()
    parent = nn.Sequential(m)
    for move in (lambda: m.to('cpu'), lambda: m.float(), lambda: parent.to('cpu'), lambda: parent.double()):
        _value(m)
        n = m.builds
        move()
        assert m.cached('w') is None
        _value(m)
        assert m.builds == n + 1


def test_forget_drops_one_entry():
    m = _Counted()
    _value(m)
    m.store('clip', 'constants', True)
    m.forget('clip')
    assert m.cached('clip', True) is None and m.cached('w') is not None
    m.forget('never stored')


def test_watched_module_changes_trigger_a_rebuild():
    m = _Counted()
    watched, unrelated = nn.Linear(3, 3), nn.Linear(3, 3)
    v = _value(m, watch=(watched,))
    with torch.no_grad():
        unrelated.weight.add_(1.0)
    unrelated.load_state_dict(nn.Linear(3, 3).state_dict())
    assert _value(m, watch=(watched,)) is v and m.builds == 1
    with torch.no_grad():                                              # an in-place edit of a watched parameter
        watched.bias.add_(1.0)
    v2 = _value(m, watch=(watched,))
    assert v2 is not v and m.builds == 2
    watched.load_state_dict(nn.Linear(3, 3).state_dict())             # a load of the watched module alone
    v3 = _value(m, watch=(watched,))
    assert v3 is not v2 and m.builds == 3
    assert _value(m, watch=(watched,)) is v3 and m.builds == 3
