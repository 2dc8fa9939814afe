"""CPU checks of the exchange matrix (tests/exchangecases.py): every map, Final and reader plan tests/test_gpu_exchange.py runs is
accepted by the planner and NVRTC-compiles for sm_90a, so a plan the encoder broke shows without a GPU; the refusals the planner
decides on its own; and the receive layout of the count matrix."""
import ctypes as C

import pytest

import exchangecases as X
from comet_b200 import proto as P


@pytest.fixture(scope="module")
def native():
    from comet_b200 import native
    return native


def supports(native, plan):
    err = native._Error()
    ok = native.lib().cb200_supports(plan, len(plan), C.byref(err))
    return bool(ok), err.code, err.message.decode(errors="replace")


@pytest.mark.parametrize("world", [1, 2, 4])
def test_every_plan_compiles(native, world):
    for plan in X.all_map_plans(world):
        ok, code, msg = supports(native, plan)
        assert ok, msg
        native.compile_plan(plan)


def test_refusals_the_planner_decides(native):
    """hash partitioning beyond 16 384 partitions or 8 keys is refused before any data arrives (the exchange's own refusals need a
    communicator: tests/test_gpu_exchange.py)"""
    types = [P.INT32] * 9
    ok, code, msg = supports(native, P.shuffle_writer(P.scan([P.INT64]), P.hash_partitioning([P.bound(0, P.INT64)], 16385)))
    assert not ok and code == 1 and "partitions" in msg
    ok, code, msg = supports(native, P.shuffle_writer(P.scan(types), P.hash_partitioning([P.bound(i, P.INT32) for i in range(9)], 2)))
    assert not ok and code == 1 and "8 hash-partition keys" in msg


def test_row_bytes():
    """one validity byte per column and row, whatever the column's NULLs"""
    c = X.e2e_case("i64", 1, n=8)
    assert X.row_bytes([P.INT64, P.DECIMAL(22, 2), P.BOOL]) == 9 + 17 + 2      # Config 4, decimal: key, sum, is_empty
    assert X.row_bytes([P.INT64, P.DOUBLE]) == 9 + 9
    assert X.row_bytes(c.state_types()) == sum(X.WIDTH[t.name] + 1 for t in c.state_types())


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_receive_layout(native, world):
    counts = [(s * 7 + p * 3) % 5 for s in range(world) for p in range(world)]
    for me in range(world):
        total, rc, ro = native.exchange_layout(counts, world, me)
        assert rc == [counts[s * world + me] for s in range(world)]
        assert ro == [sum(rc[:s]) for s in range(world)] and total == sum(rc)
