"""CPU: the fused renderer's mbarrier and bulk-copy protocol at the ring sizes render_fused_ws3.cu builds with.

tests/test_fused_protocol_sim_cpu.py simulates the protocol with a 4-stage A1 ring and 3 colour tiles in shared memory.
The kernel now holds one A1 stage per gather team (kNA = 3) and two colour tiles (kColBufs = 2), so that its shared memory
fits the 196 KB carve-out and leaves 60 KB of L1 to the gather.  This file runs the same simulation - the same role
transcriptions, hazard checks and negative controls - at the sizes read from the kernel source, so the simulated ring
depths cannot drift from the built ones."""
import os
import re

import pytest

from tests import test_fused_protocol_sim_cpu as sim

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'panic3d-anime-reconstruction_b200', 'csrc', 'render_fused_ws3.cu')


def _kernel_constant(name):
    with open(SRC) as f:
        m = re.search(r'constexpr int %s = (\d+);' % name, f.read())
    assert m, f'{name} not found in render_fused_ws3.cu'
    return int(m.group(1))


K_NA, K_COL_BUFS = _kernel_constant('kNA'), _kernel_constant('kColBufs')


@pytest.fixture
def kernel_rings(monkeypatch):
    monkeypatch.setattr(sim, 'K_NA', K_NA)
    monkeypatch.setattr(sim, 'K_COL_BUFS', K_COL_BUFS)


def test_ring_sizes_are_the_kernels():
    assert (K_NA, K_COL_BUFS) == (3, 2)
    assert 6 % K_COL_BUFS == 0          # colours() walks a group's six tiles through the buffers in whole rounds


@pytest.mark.parametrize('N', [1, 2, 3, 4, 5, 7, 8, 13])
def test_protocol_has_no_deadlock_or_hazard(N, kernel_rings):
    for seed in [s * 101 + N for s in range(12)] + [s * 131 + N for s in range(1, 13)]:
        sim.Sim(N, seed).run()


@pytest.mark.parametrize('kw, match', [
    (dict(sig_count=4), 'sigma was stored'),
    (dict(first_wait='read'), 'issued before its store completed'),
    (dict(staging_wait=False), 'rewritten before its bulk store read it'),
    (dict(colours_k=1), 'overwritten before its load completed'),
])
def test_simulation_still_catches_each_protocol_bug(kw, match, kernel_rings):
    """The negative controls of the 4 / 3 simulation, at 3 / 2: each missing wait is still caught."""
    with pytest.raises(AssertionError, match=match):
        for seed in range(40):
            sim.Sim(4, seed, **kw).run()
