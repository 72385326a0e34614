"""The unicast shared areas give their device memory back: the two-shot's gather area, the LL, ring and push areas,
and the all-to-all's exchange area.  Open, one call of each measurement that builds one, and close leave free memory
where it was, at N = 1 and with three ranks on one device; on an open handle, a second round of the same calls
allocates nothing more.

The domains are single-process: each process's reading of free memory would include whatever another process holds at
that moment, and nothing synchronises two processes after close.  The multi-process suites cover the import and release
path by passing."""
import pytest

pytestmark = pytest.mark.gpu

SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
NBYTES = 64 << 20  # bytes_per_pair: an area left behind holds at least 2 MiB per rank, most of them 64 MiB or more


def free_bytes():
    import torch
    torch.cuda.synchronize(0)
    return torch.cuda.mem_get_info(0)[0]


def open_ranks(pkg, n):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=NBYTES, flags=SAME if n > 1 else 0, ctas=8, timeout_ms=20000))


def call_each(p, n):
    """One call of every measurement with a unicast shared area; each must run on every rank, or it built nothing."""
    for fn in (p.AllReduceTwoShot, p.AllReduceLL, p.AllReduceRing, p.AllReducePush, p.AllToAll):
        out = fn(reps=1)
        assert out.measured == [True] * n and out.status == [0] * n, (fn.__name__, out.status)


@pytest.mark.parametrize("n", [1, 3])
def test_open_calls_and_close_give_back_the_device_memory(pkg, n):
    def cycle():
        with open_ranks(pkg, n) as p:
            call_each(p, n)
    cycle()  # the first cycle loads the kernels
    start = free_bytes()
    for _ in range(2):
        cycle()
    assert free_bytes() >= start - (2 << 20)


@pytest.mark.parametrize("n", [1, 3])
def test_a_second_round_on_an_open_handle_allocates_nothing(pkg, n):
    with open_ranks(pkg, n) as p:
        call_each(p, n)
        before = free_bytes()
        call_each(p, n)
        assert free_bytes() == before
