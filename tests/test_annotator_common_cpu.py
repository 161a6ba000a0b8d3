"""The annotators' shared size-keyed table cache (ctrlora_b200/annotator/common.py SizeCache): bounded, least recently
used first out, and rebuilt when a parameter it was built from changes in place."""
import torch

from ctrlora_b200.annotator.common import SizeCache


def test_size_cache_bounded_lru_and_rebuilt_on_parameter_change():
    p = torch.nn.Parameter(torch.zeros(3), requires_grad=False)
    builds = []

    def fetch(cache, key):
        def build():
            builds.append(key)
            return p.detach().clone() + key
        return cache.fetch(key, build, [p])

    cache = SizeCache(3)
    for key in (1, 2, 3):
        fetch(cache, key)
    first = fetch(cache, 1)                        # a hit: no build, and 1 is now the most recently used
    assert builds == [1, 2, 3] and first is cache[1]
    fetch(cache, 4)                                # evicts 2, the least recently used
    assert list(cache) == [3, 1, 4] and len(cache) == 3
    fetch(cache, 2)                                # evicts 3
    assert list(cache) == [1, 4, 2] and builds == [1, 2, 3, 4, 2]

    p.add_(10.0)                                   # in place, as load_state_dict writes: the version moves
    rebuilt = fetch(cache, 1)
    assert builds[-1] == 1 and rebuilt is not first
    assert torch.equal(rebuilt, torch.full((3,), 11.0))
    assert list(cache) == [4, 2, 1] and len(cache) == 3
