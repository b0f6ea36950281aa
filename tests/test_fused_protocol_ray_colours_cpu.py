"""CPU: discrete-event simulation of the fused renderer's protocol as csrc/render_fused_ws3.cu builds it now, with each
group's colour reduction (colours()) on the RAY warps.  tests/test_fused_protocol_sim_cpu.py models the previous protocol,
in which the decoder ran colours(); this file reuses its barriers, bulk-copy delays and scheduler, and transcribes the
three roles of the current kernel:
  * decoder: after a group's fine pass is stored, the elected thread of each warpgroup waits for its bulk stores to complete
    and arrives on col_stored[n & 1] (in the next tile's epilogue, and after the tile loop for the last group); before the
    first store into a colour area it waits for the state_free of the area's previous group (CA[m % 3]: m - 3, FA[m & 1]:
    m - 2);
  * ray warp: after composite(n) it waits on col_stored, bulk-loads only its own rays' rows of each tile into col_buf
    (its own col_full barriers), reloads a buffer once it has read it, and arrives on state_free[n & 3] (count 4).
Rows are tracked in 16-row blocks: warpgroup h stores blocks 4h .. 4h + 3 of a tile, ray warp rw loads blocks 2rw, 2rw + 1
(S = 96) or rw, rw + 4 (S = 48).  Asserted, over many seeds and group counts:
  * no deadlock and no lost mbarrier phase, and every group's colours are reduced by all four ray warps;
  * a ray warp's load is issued only after col_stored fired for its group and the stores of its blocks completed;
  * a col_buf buffer is reloaded only after its warp read it, and read only after its load landed;
  * CA / FA blocks are not overwritten before the previous group's loads of them landed;
  * and the checks of the previous model that still apply: the A1 ring, the sigma hand-off, the per-group state slot and
    the staging tile.
The negative controls at the end drop one wait each and must fail with their own message."""
import pytest

from tests import test_fused_protocol_sim_cpu as base
from tests.test_fused_protocol_rings_cpu import K_COL_BUFS, K_NA
from tests.test_fused_protocol_sim_cpu import Bar, TxBar, pass_at, tile_at

K_EW, K_RW, K_TEAMS = base.K_EW, base.K_RW, base.K_TEAMS


class RayColoursSim(base.Sim):
    def __init__(self, N, seed, S=96, col_stored_wait=True, coarse_guard=True, fine_guard=True, fine_areas=2,
                 reload_after_read=True):
        # The kernel's choices; the other values model bugs that the negative controls below must catch:
        #   col_stored_wait    the ray warps wait on col_stored before their first loads of a group
        #   coarse_guard       the decoder waits for state_free of group m - 3 before its first store into CA[m % 3]
        #   fine_guard         ... of group m - 2 before its first store into FA[m % fine_areas]
        #   fine_areas         fine colour areas (2: FA[n & 1])
        #   reload_after_read  a ray warp reloads a buffer after reading it (else right after its col_full wait)
        super().__init__(N, seed)
        self.S, self.col_stored_wait, self.reload_after_read = S, col_stored_wait, reload_after_read
        self.coarse_guard, self.fine_guard, self.fine_areas = coarse_guard, fine_guard, fine_areas
        self.a1_full = [Bar(4) for _ in range(K_NA)]; self.a1_empty = [Bar(K_EW) for _ in range(K_NA)]
        self.a1_tile, self.a1_written, self.a1_read = [None] * K_NA, [0] * K_NA, [0] * K_NA
        self.state_free = [Bar(K_RW) for _ in range(4)]
        self.col_stored = [Bar(2) for _ in range(2)]
        self.col_full = [[TxBar(1) for _ in range(K_COL_BUFS)] for _ in range(K_RW)]
        self.col_signalled = set()                    # groups whose col_stored phase completed
        self.area_content = {}                        # (area, block) -> (group, tile) whose store completed there
        self.area_last = {}                           # (area, block) -> (group, tile) last stored there
        self.load_done = set()                        # (group, tile, block) whose load landed
        self.buf = [[None] * K_COL_BUFS for _ in range(K_RW)]          # [warp][b] -> (group, tile, landed?)
        self.buf_read = [[False] * K_COL_BUFS for _ in range(K_RW)]
        self.colours_warps = {}                       # group -> ray warps that finished its colours

    def area(self, n, p, k):
        return ('CA', n % 3, k) if p == 0 else ('FA', n % self.fine_areas, k)

    def blocks(self, rw):
        return (2 * rw, 2 * rw + 1) if self.S == 96 else (rw, rw + K_RW)

    # ---------------------------------------------------------------- bulk copies
    def bulk_store(self, h, n, p, k):                # elected thread of warpgroup h: blocks 4h .. 4h + 3 of tile k
        area = self.area(n, p, k)
        kind = 'coarse' if p == 0 else 'fine'
        for blk in range(4 * h, 4 * h + 4):
            prev = self.area_last.get((area, blk))
            if prev is not None:
                m, t = prev
                assert (m, t, blk) in self.load_done, f'{kind} area {area} block {blk} of group {m} overwritten before its load landed'
            self.area_last[(area, blk)] = (n, 3 * p + k)
        rec = {'read': False, 'all': False}
        self.bulk_groups[h].append(rec)
        t_read = self.dur(0.05, 1.0) if self.rng.random() < 0.9 else self.dur(1.0, 20.0)
        self.later(t_read, lambda: rec.__setitem__('read', True))

        def written():
            rec['all'] = True
            for blk in range(4 * h, 4 * h + 4):
                self.area_content[(area, blk)] = (n, 3 * p + k)
        self.later(t_read + (self.dur(0.05, 4.0) if self.rng.random() < 0.9 else self.dur(4.0, 40.0)), written)

    def ray_load(self, rw, n, t):                    # lane 0 of ray warp rw: its blocks of tile t into col_buf[t % 2]
        p, k = divmod(t, 3)
        b, area = t % K_COL_BUFS, self.area(n, p, k)
        blocks = self.blocks(rw)
        assert n in self.col_signalled and all(self.area_content.get((area, blk)) == (n, t) for blk in blocks), \
            f'load of {area} for group {n} (warp {rw}) issued before col_stored signalled its completed stores'
        assert self.buf[rw][b] is None or self.buf_read[rw][b], f'col_buf[{b}] rows of warp {rw} reloaded before it read them'
        self.col_full[rw][b].arrive_expect_tx()
        self.buf[rw][b], self.buf_read[rw][b] = (n, t, False), False

        def landed():
            self.buf[rw][b] = (n, t, True)
            for blk in blocks:
                self.load_done.add((n, t, blk))
            self.col_full[rw][b].complete_tx()
        self.later(self.dur(0.2, 3.0) if self.rng.random() < 0.9 else self.dur(3.0, 30.0), landed)

    # ---------------------------------------------------------------- roles
    def gather_warp(self, gw):
        team, it = gw >> 2, 0
        for q in range(self.T):
            n, p, k = tile_at(q, self.N)
            my_it = it; it += 1
            if my_it % K_TEAMS != team:
                continue
            if p == 0:
                yield ('wait', self.state_free[n & 3], ((n >> 2) & 1) ^ 1)
                prev = self.state_owner[n & 3]
                assert prev is None or prev == n or prev in self.colours_done, f'state slot of group {prev} rewritten for {n}'
                self.state_owner[n & 3] = n
            else:
                yield ('wait', self.fine_ready[n & 3], (n >> 2) & 1)
                assert n in self.importance_done, f'fine gather of {n} before its importance sampling'
            stage = my_it % K_NA
            yield ('wait', self.a1_empty[stage], ((my_it // K_NA) & 1) ^ 1)
            if self.a1_tile[stage] != q:
                assert self.a1_tile[stage] is None or self.a1_read[stage] == K_EW, f'A1 stage {stage} rewritten before it was read'
                self.a1_tile[stage], self.a1_written[stage], self.a1_read[stage] = q, 0, 0
            yield ('work', self.dur(5, 20))
            self.a1_written[stage] += 1
            self.a1_full[stage].arrive()

    def decoder_warp(self, e):
        h, elect = e >> 2, (e & 3) == 0
        mark = {'stored': -1, 'signalled': -1}

        def signal_stored():
            if elect:
                yield from self.bulk_wait(h, 'all')
                bar, n = self.col_stored[mark['stored'] & 1], mark['stored']
                phase = bar.phase
                bar.arrive()
                if bar.phase != phase:
                    self.col_signalled.add(n)
            mark['signalled'] = mark['stored']

        for it in range(self.T):
            n, p, k = tile_at(it, self.N)
            stage = it % K_NA
            yield ('wait', self.a1_full[stage], (it // K_NA) & 1)
            assert self.a1_tile[stage] == it and self.a1_written[stage] == 4, f'decoder reads A1 stage {stage} before tile {it} is complete'
            yield ('work', self.dur(0.5, 2))          # layer 1
            self.a1_read[stage] += 1
            self.a1_empty[stage].arrive()
            yield ('work', self.dur(1, 4))            # softplus, layer 2
            if mark['stored'] > mark['signalled']:
                yield from signal_stored()
            elif elect:
                yield from self.bulk_wait(h, 'read')
            yield ('wgbar', h)
            assert all(r['read'] for r in self.bulk_groups[h]), f'staging of warpgroup {h} rewritten before its bulk store read it'
            yield ('work', self.dur(0.2, 1))          # staging and sigma stores
            self.sigma_writes[(n, p)] = self.sigma_writes.get((n, p), 0) + 1
            yield ('wgbar', h)
            if elect:
                prev = n - (3 if p == 0 else 2)
                if k == 0 and prev >= 0 and (self.coarse_guard if p == 0 else self.fine_guard):
                    yield ('wait', self.state_free[prev & 3], (prev >> 2) & 1)
                self.bulk_store(h, n, p, k)
            if k == 2:
                if p == 1:
                    mark['stored'] = n
                (self.sigc_ready if p == 0 else self.sigf_ready)[n & 3].arrive()
        yield from signal_stored()

    def colours(self, rw, n):
        if self.col_stored_wait:
            yield ('wait', self.col_stored[n & 1], (n >> 1) & 1)
        for t in range(K_COL_BUFS):
            self.ray_load(rw, n, t)
        for t in range(6):
            b = t % K_COL_BUFS
            yield ('wait', self.col_full[rw][b], ((6 * n + t) // K_COL_BUFS) & 1)
            assert self.buf[rw][b] == (n, t, True), f'colours({n}) of warp {rw} reads col_buf[{b}] before tile {t} landed'
            if not self.reload_after_read and t + K_COL_BUFS < 6:
                self.ray_load(rw, n, t + K_COL_BUFS)
            yield ('work', self.dur(0.2, 1.5))
            assert self.buf[rw][b] == (n, t, True), f'col_buf[{b}] of warp {rw} changed while colours({n}) read it'
            self.buf_read[rw][b] = True
            if self.reload_after_read and t + K_COL_BUFS < 6:
                self.ray_load(rw, n, t + K_COL_BUFS)
        yield ('work', self.dur(0.1, 0.5))            # the warp's out_rgb rows

    def ray_warp(self, rw):
        for j in range(2 * self.N):
            n, p = pass_at(j, self.N)
            si, par = n & 3, (n >> 2) & 1
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
                yield ('work', self.dur(2, 12))       # composite: omega / pos of the warp's own rays
                if rw == 0:
                    self.composite_done.add(n)
                yield from self.colours(rw, n)
                self.colours_warps[n] = self.colours_warps.get(n, 0) + 1
                if self.colours_warps[n] == K_RW:
                    self.colours_done.add(n)
                self.state_free[si].arrive()


def _seeds(N):
    return [s * 101 + N for s in range(12)] + [s * 131 + N for s in range(1, 13)]


@pytest.mark.parametrize('S', [96, 48])
@pytest.mark.parametrize('N', [1, 2, 3, 4, 5, 7, 8, 13])
def test_protocol_has_no_deadlock_or_hazard(N, S):
    for seed in _seeds(N):
        RayColoursSim(N, seed, S=S).run()


@pytest.mark.parametrize('kw, match', [
    # without the col_stored wait, a ray warp loads colours whose stores have not completed
    (dict(col_stored_wait=False), 'issued before col_stored signalled its completed stores'),
    # without the coarse area's guard, C(m) overwrites CA[m % 3] while group m - 3's loads may be in flight
    (dict(coarse_guard=False), r'coarse area .* overwritten before its load landed'),
    # a reload issued right after the col_full wait overwrites rows the warp has not read
    (dict(reload_after_read=False), 'reloaded before it read them'),
    # with a single fine area and no guard, F(m + 1) overwrites it while group m's loads may be in flight
    (dict(fine_areas=1, fine_guard=False), r"fine area \('FA', 0, \d\) .* overwritten before its load landed"),
])
@pytest.mark.parametrize('S', [96, 48])
def test_simulation_catches_each_protocol_bug(kw, match, S):
    # the coarse areas have about five tiles of slack, so their hazard needs a long bulk-copy tail: up to 200 seeds
    with pytest.raises(AssertionError, match=match):
        for seed in range(200):
            RayColoursSim(13, seed, S=S, **kw).run()
