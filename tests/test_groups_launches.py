"""Kernel launches of one hs_verify_groups call with a registered committee: a fixed count per call, with and without verdict modes."""
import numpy as np
import pytest

from test_groups_dev import _clear, _register, expected, keys, make_burst, run_host  # noqa: F401 (keys is a fixture)


@pytest.mark.gpu
@pytest.mark.parametrize("indexed, launches", [(False, 6), (True, 4)])
def test_verify_groups_launch_count(engine, oracle, keys, indexed, launches):
    """Digest, lookup, miss pass, main, finish and the group AND with key bytes (one key outside the committee); digest, main, finish
    and the group AND in the committee-indexed form.  The verdicts equal the oracle's."""
    rng = np.random.default_rng(606)
    b = make_burst(oracle, keys, rng, 700, foreign=not indexed)
    _register(engine, keys)
    try:
        for modes in (True, False):
            want_g, want_i = expected(oracle, keys, b, indexed, modes)
            l0 = engine.kernel_launches
            g, items = run_host(engine, b, indexed, modes)
            assert engine.kernel_launches - l0 == launches, modes
            assert (items == want_i).all() and (g == want_g).all()
    finally:
        _clear(engine)
