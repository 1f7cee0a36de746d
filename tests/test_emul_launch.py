"""CPU tests of the warp emulator's launch entry point (tests/emul/emul_main.cpp): its ctypes mirror of RolloutArgs
matches the C++ layout, and its restatement of rollout_kernel's prologue maps CTAs to rows as the kernel does."""
import ctypes as C

import numpy as np
import pytest

from tests.emul import emul


@pytest.fixture(scope="module")
def lib():
    return emul.build()


def test_rollout_args_layout(lib):
    """emul.build checks every field offset and the size at load; the walk here pins that the check sees them all."""
    off, names, i = C.c_size_t(), [], 0
    while (name := lib.emul_rollout_field(i, C.byref(off))) is not None:
        assert emul.RolloutArgs._fields_[i][0] == name.decode()
        assert getattr(emul.RolloutArgs, name.decode()).offset == off.value
        names.append(name.decode())
        i += 1
    assert names == [f for f, _ in emul.RolloutArgs._fields_]
    assert off.value == C.sizeof(emul.RolloutArgs)


@pytest.mark.parametrize("nrows, rpi, rpm, models", [(7, 0, 0, False), (40, 0, 0, False)] + [
    (n, rpi, rpm, models) for n, rpi, rpm in ((3 * 17, 17, 0), (4 * 33, 33, 0), (2 * 3 * 9, 3 * 9, 9),
                                              (5 * 2 * 65, 2 * 65, 65)) for models in (False, True)])
def test_every_row_runs_once_on_its_slot(lib, nrows, rpi, rpm, models):
    """For wpc 1..16, with and without iteration limits: every row of a running instance is run by exactly one
    active warp, every CTA stages the slot cta_instance names, and the grid is launch_rollout's."""
    rps = rpm if rpm > 0 else rpi
    B = nrows // rpi if rpi else 1
    lims = [None] if models is False and rpi == 0 else [None, np.array([(b % 3) for b in range(B)], np.int32)]
    for wpc in range(1, 17):
        for lim in lims:
            A = emul.RolloutArgs(nrows=nrows, rows_per_inst=rpi, rows_per_model=rpm if models else 0, iter=1)
            if lim is not None:
                if not models and rpi % wpc:
                    continue   # the host launches instance-aligned CTAs whenever limits are set
                A.iter_lim = lim.ctypes.data
            grid = (nrows // rps) * -(-rps // wpc) if models else -(-nrows // wpc)
            staged, runs = np.full(grid, -7, np.int32), np.zeros(nrows, np.int32)
            n_slots = nrows // rps if models else 1
            assert lib.emul_launch_map(C.byref(A), int(models), n_slots, wpc, staged.ctypes.data,
                                       runs.ctypes.data) == grid, wpc
            inst = np.arange(nrows) // rpi if rpi else np.zeros(nrows, int)
            want = np.ones(nrows, np.int32) if lim is None else (1 < lim[inst]).astype(np.int32)
            assert np.array_equal(runs, want), (wpc, lim)
            for cta in range(grid):
                ci = lib.emul_cta_instance(nrows, rpi, rpm if models else 0, int(models), cta, wpc)
                if lim is not None and not 1 < lim[ci]:
                    assert staged[cta] == -1, (wpc, cta)
                elif models:
                    assert staged[cta] >= 0 and staged[cta] * rps // rpi == ci, (wpc, cta)
                else:
                    assert staged[cta] == 0, (wpc, cta)
