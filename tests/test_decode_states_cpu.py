"""generate()'s decode-state cache (navillm_b200.generation.DecodeStates): lookup-or-build, least-recently-used eviction, no
caching without a graph, clear()."""
from navillm_b200.generation import DecodeStates


def _builder(built):
    def build(name):
        def make():
            built.append(name)
            return {"name": name}
        return make
    return build


def test_a_hit_returns_the_cached_state_and_moves_it_to_the_end():
    built = []
    build = _builder(built)
    states = DecodeStates()
    a = states.lookup("a", build("a"), True)
    states.lookup("b", build("b"), True)
    assert list(states) == ["a", "b"]
    assert states.lookup("a", build("a again"), True) is a
    assert built == ["a", "b"] and list(states) == ["b", "a"]


def test_the_least_recently_used_state_is_evicted_at_the_limit():
    built = []
    build = _builder(built)
    states = DecodeStates()
    assert states.max_states == 2
    states.lookup("a", build("a"), True)
    states.lookup("b", build("b"), True)
    states.lookup("a", build("a"), True)                  # a is now the most recently used
    states.lookup("c", build("c"), True)
    assert list(states) == ["a", "c"]
    states.lookup("b", build("b"), True)                  # b was evicted: built again
    assert built == ["a", "b", "c", "b"] and list(states) == ["c", "b"]
    states.max_states = 3
    states.lookup("d", build("d"), True)
    assert list(states) == ["c", "b", "d"]


def test_nothing_is_cached_without_a_graph():
    built = []
    build = _builder(built)
    states = DecodeStates()
    a = states.lookup("a", build("a"), True)
    e1 = states.lookup("a", build("eager"), False)        # an eager call neither reads nor writes the cache
    e2 = states.lookup("x", build("eager x"), False)
    assert e1 is not a and e2 is not e1
    assert built == ["a", "eager", "eager x"] and list(states) == ["a"]


def test_clear_drops_every_state():
    built = []
    build = _builder(built)
    states = DecodeStates()
    states.lookup("a", build("a"), True)
    states.lookup("b", build("b"), True)
    states.clear()
    assert len(states) == 0
    states.lookup("a", build("a"), True)
    assert built == ["a", "b", "a"]
