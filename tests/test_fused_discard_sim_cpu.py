"""CPU: the fused renderer's L2 line discards in the protocol simulation of tests/test_fused_protocol_sim_cpu.py.

Once a ray warp's bulk load of its rows of a colour tile has landed, its lanes discard those rows' lines from L2
(discard.global.L2: the lines leave L2 without a write-back, their contents become undefined).  A discard is a generic-proxy
write, so it must be ordered before the decoder's next bulk store (async proxy) into the same lines, or the store's colours
could be dropped.  The kernel orders it through the state_free hand-off the stores already wait for: the warp discards
before lane 0 arrives on state_free (release), and the decoder's elected thread issues fence.proxy.async.global after its
state_free wait (acquire) and before the store.  This module adds the discard to the simulation as an event:
  * a ray warp discards its rows of tile t after its col_full wait, and its discards of group n are released when it
    arrives on state_free for n;
  * a bulk store into an area fails if a discard of any of its rows is still pending (not released);
  * a discard issued after the next store into its rows fails the same way.
The negative control moves the discards after the arrive and must fail at S = 96 and at S = 48.  The simulation itself
(roles, barriers, bulk copies and their checks) is the one of tests/test_fused_protocol_sim_cpu.py, imported unchanged."""
import os
import re

import pytest

from panic3d_b200 import _build
from tests.test_fused_protocol_sim_cpu import K_COL_BUFS, K_EW, K_RW, K_STATES, Sim, pass_at

with open(os.path.join(_build.CSRC, 'render_fused_ws3.cu')) as _f:
    SRC = _f.read()


class DiscardSim(Sim):
    def __init__(self, N, seed, S=96, discard='before_arrive', **kw):
        # discard: 'before_arrive' (the kernel) | 'after_arrive' (the negative control)
        super().__init__(N, seed, S=S, **kw)
        self.discard = discard
        self.discards = {}                           # (area, block) -> {'group', 'released'} of its last discard
        self.discard_count = 0

    def issue_discards(self, rw, n, t):
        p, k = divmod(t, 3)
        area = self.area(n, p, k)
        for blk in self.blocks(rw):
            last = self.area_last.get((area, blk))
            assert last is not None and last[0] == n, \
                f'discard of {area} block {blk} (group {n}) still pending when the store of group {last[0]} was issued'
            self.discards[(area, blk)] = {'group': n, 'warp': rw, 'released': False}
            self.discard_count += 1

    def release_discards(self, rw, n):               # lane 0's arrive on state_free (release) after the warp's discards
        for d in self.discards.values():
            if d['group'] == n and d['warp'] == rw:
                d['released'] = True

    def bulk_store(self, h, n, p, k):
        area = self.area(n, p, k)
        for blk in range(4 * h, 4 * h + 4):
            d = self.discards.get((area, blk))
            assert d is None or d['released'], \
                f'discard of {area} block {blk} (group {d["group"]}) still pending when the store of group {n} was issued'
        super().bulk_store(h, n, p, k)

    def colours(self, rw, n):                        # Sim.colours with the discard after each col_full wait
        if self.col_stored_wait:
            yield ('wait', self.col_stored[n & 1], (n >> 1) & 1)
        for t in range(K_COL_BUFS):
            self.ray_load(rw, n, t)
        for t in range(6):
            b = t % K_COL_BUFS
            yield ('wait', self.col_full[rw][b], ((6 * n + t) // K_COL_BUFS) & 1)
            assert self.buf[rw][b] == (n, t, True), f'colours({n}) of warp {rw} reads col_buf[{b}] before tile {t} landed'
            if self.discard == 'before_arrive':
                self.issue_discards(rw, n, t)
            yield ('work', self.dur(0.2, 1.5))
            assert self.buf[rw][b] == (n, t, True), f'col_buf[{b}] of warp {rw} changed while colours({n}) read it'
            self.buf_read[rw][b] = True
            if t + K_COL_BUFS < 6:
                self.ray_load(rw, n, t + K_COL_BUFS)
        yield ('work', self.dur(0.1, 0.5))

    def ray_warp(self, rw):                          # Sim.ray_warp's fine-pass branch with the release / the late discards
        for j in range(2 * self.N):
            n, p = pass_at(j, self.N)
            si, par = n % K_STATES, (n // K_STATES) & 1
            if p == 0:
                yield ('wait', self.sigc_ready[si], par)
                assert self.sigma_writes.get((n, 0), 0) == 3 * K_EW, f'importance({n}) before every coarse sigma was stored'
                yield ('work', self.dur(2, 12))
                if rw == 0:
                    self.importance_done.add(n)
                self.fine_ready[si].arrive()
            else:
                yield ('wait', self.sigf_ready[si], par)
                assert self.sigma_writes.get((n, 1), 0) == 3 * K_EW, f'composite({n}) before every fine sigma was stored'
                yield ('work', self.dur(2, 12))
                yield from self.colours(rw, n)
                self.colours_warps[n] = self.colours_warps.get(n, 0) + 1
                if self.colours_warps[n] == K_RW:
                    self.colours_done.add(n)
                if self.discard == 'before_arrive':
                    self.release_discards(rw, n)
                self.state_free[si].arrive()
                if self.discard == 'after_arrive':
                    yield ('work', self.dur(0.0, 2.0))
                    for t in range(6):
                        self.issue_discards(rw, n, t)


def test_kernel_fences_between_state_free_and_the_store():
    """The decoder's elected thread: state_free wait, then fence.proxy.async.global, then the bulk store into the area."""
    m = re.search(r'RC_WAIT\(1, RC_STATE_FREE, &sm\.state_free\[prev & 3\], \(prev >> 2\) & 1\);\s*'
                  r'fence_proxy_async_global\(\);\s*\}\s*bulk_store\(colour_area', SRC)
    assert m, 'fence.proxy.async.global must follow the state_free wait and precede the bulk store into the colour area'
    # the ray warp: discards inside colours(), a __syncwarp, then lane 0's arrive on state_free
    assert re.search(r'colours\(n, back\);\s*__syncwarp\(\);[^\n]*\n\s*if \(lane == 0\) mbar_arrive\(&sm\.state_free\[si\]\);', SRC)
    assert SRC.count('l2_discard_line(') == 1


@pytest.mark.parametrize('S', [96, 48])
@pytest.mark.parametrize('N', [1, 2, 3, 5, 8, 13])
def test_discards_are_released_before_the_next_store(N, S):
    for seed in [s * 101 + N for s in range(8)]:
        sim = DiscardSim(N, seed, S=S)
        sim.run()
        assert sim.discard_count == N * 6 * K_RW * 2                # every row block of every tile, once
        assert all(d['released'] for d in sim.discards.values())


@pytest.mark.parametrize('S', [96, 48])
def test_simulation_catches_a_discard_after_the_arrive(S):
    with pytest.raises(AssertionError, match=r'discard of .* still pending when the store of group \d+ was issued'):
        for seed in range(200):
            DiscardSim(13, seed, S=S, discard='after_arrive').run()
