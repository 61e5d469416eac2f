"""PreparedMixin: one cache for the values a module derives from its parameters (folded and packed weights, per-clip constants).

Every entry is dropped when the module, or any module above it, loads a state_dict or is moved or cast (`.to()`, `.cuda()`, `.float()`):
nn.Module runs `_load_from_state_dict` and `_apply` for every module of the tree.  A hit costs one dict lookup."""
from __future__ import annotations

import itertools


class PreparedMixin:
    """Mix in before nn.Module: `class M(PreparedMixin, nn.Module)`."""

    def __init__(self):
        super().__init__()
        self._prep_entries = {}

    def prepared(self, name, build, *key, watch=()):
        """The value cached as `name` for `key` (e.g. the split flag); `build()` makes it on a miss and replaces the value of any other key.
        watch: modules whose parameters' and buffers' (data_ptr, _version) are part of the key, for modules the caller owns and may load or
        edit on their own (the torso warper)."""
        if watch:
            key += (tuple((t.data_ptr(), t._version) for m in watch for t in itertools.chain(m.parameters(), m.buffers())),)
        hit = self._prep_entries.get(name)
        if hit is None or hit[0] != key:
            hit = self._prep_entries[name] = (key, build())
        return hit[1]

    def cached(self, name, *key):
        """The value cached as `name` for `key`, or None; builds nothing."""
        hit = self._prep_entries.get(name)
        return hit[1] if hit is not None and hit[0] == key else None

    def store(self, name, value, *key):
        """Cache `value` as `name` for `key` (values made outside `prepared`, such as a clip's constants) and return it."""
        self._prep_entries[name] = (key, value)
        return value

    def forget(self, name) -> None:
        self._prep_entries.pop(name, None)

    def _load_from_state_dict(self, *a, **k):
        self._prep_entries.clear()
        return super()._load_from_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self._prep_entries.clear()
        return super()._apply(fn, *a, **k)
