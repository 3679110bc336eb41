"""Launch sites of the engine's ring and load-generation kernels.  In hs_engine.cu each of them is launched from one function, which the
latency path, the verify queue and hs_self_test all call, so the self-test runs the launches the product runs.  The ring those kernels
work over is allocated by one function."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE = os.path.join(ROOT, "hotstuff_b200", "csrc", "hs_engine.cu")
ONE_LAUNCH = ("k_verify_small", "k_verify_bulk", "k_queue_generic", "k_queue_digests", "k_digest32_long", "k_keygen", "k_sign_digests")
LAUNCH = re.compile(r"\b(k_\w+)\s*(?:<[^<>;]*>)?\s*<<<")


def _code():
    """hs_engine.cu without comments and string literals."""
    with open(ENGINE) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    return "\n".join(re.sub(r'"(\\.|[^"\\])*"', '""', s).split("//", 1)[0] for s in src.splitlines())


def test_each_ring_and_load_generation_kernel_has_one_launch():
    launches = [m.group(1) for m in LAUNCH.finditer(_code())]
    counts = {k: launches.count(k) for k in ONE_LAUNCH}
    assert counts == {k: 1 for k in ONE_LAUNCH}, counts


def test_ring_records_are_allocated_at_one_site():
    code = _code()
    allocs = re.findall(r"\balloc\([^;]*sizeof\(small_rec\)", code)
    holders = re.findall(r"\bmapped<small_rec>", code)
    assert len(allocs) == 1, allocs
    assert len(holders) == 1, holders
