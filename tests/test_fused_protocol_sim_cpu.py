"""CPU: discrete-event simulation of the mbarrier and bulk-copy protocol of the fused renderer (csrc/render_fused_ws3.cu)
as it is built: its pass schedule and the hand-off between its 24 warps - 12 gather, 8 decoder (two wgmma warpgroups), 4 ray.
Every role's control flow is transcribed from the CUDA source (same loops, barriers, parities and arrival counts, the
decoder's elected threads with their bulk stores, .read and full waits, each ray warp's colours() with its own bulk loads);
the ring sizes and arrival counts are read from the source, so a change there fails here until the model follows.  Work
items get random durations and the runnable warps are stepped in random order, over many seeds and group counts, at S = 96
and 48.  Bulk copies run asynchronously with random read / write / landing delays, each with a tail longer than a tile, so
that a check fires whenever the wait guarding it is missing (the negative controls at the end).  Rows of the colour path
are tracked in 16-row blocks: warpgroup h stores blocks 4h .. 4h + 3 of a tile, ray warp rw loads blocks 2rw, 2rw + 1
(S = 96) or rw, rw + 4 (S = 48).  Asserted:
  * no deadlock and no lost mbarrier phase (a waiter that a barrier overtakes by two phases blocks forever), and every
    group's colours are reduced by all four ray warps;
  * A1 ring: the gather rewrites a stage only after all eight decoder warps have read its previous tile, and a decoder warp
    reads a stage only once all four warps of the team have written it;
  * shared-memory hazards: the ray warps read a pass's sigma only after every decoder warp wrote its rows, a per-group state
    slot is not rewritten by the gather before its previous group is finished, fine depths are read only after importance;
  * colour path: a warpgroup's staging tile is not rewritten before its last bulk store has read it; a ray warp loads a
    group's rows only after col_stored fired for the group and the bulk stores of those rows completed; it reads a col_buf
    tile only after its load landed and reloads it only after reading it; CA[n % 3] and FA[n & 1] blocks are not rewritten
    before the previous group's loads of them landed.
It mirrors the protocol, not the arithmetic; parity on hardware is what tests/test_render_gpu.py is for."""
import heapq
import os
import random
import re

import pytest

from panic3d_b200 import _build

with open(os.path.join(_build.CSRC, 'render_fused_ws3.cu')) as _f:
    SRC = _f.read()


def _kernel_constant(name):
    m = re.search(r'\bconstexpr int (?:\w+ = \d+, )*%s = (\d+)[,;]' % name, SRC)
    assert m, f'{name} not found in render_fused_ws3.cu'
    return int(m.group(1))


K_GW, K_EW, K_RW, K_TEAMS, K_NA, K_STATES, K_COL_BUFS = (
    _kernel_constant(n) for n in ('kGW', 'kEW', 'kRW', 'kTeams', 'kNA', 'kStates', 'kColBufs'))

# arrivals per phase of each mbarrier, as the roles below make them
ARRIVALS = {
    'a1_full': K_GW // K_TEAMS,                          # every warp of the gather team
    'a1_empty': K_EW, 'sigc_ready': K_EW, 'sigf_ready': K_EW,          # every decoder warp
    'fine_ready': K_RW, 'state_free': K_RW,              # every ray warp
    'col_stored': K_EW // 4,                             # the elected thread of each decoder warpgroup
    'col_full': 1,                                       # lane 0 of its ray warp, with the bytes of its bulk loads
}


def _mbar_init_counts():
    """{barrier: arrival count} of the kernel's mbar_init(&sm.<barrier>..., <count>) lines."""
    counts = {}
    for name, count in re.findall(r'mbar_init\(&sm\.(\w+)(?:\[\w+\])*, (\w+)\)', SRC):
        counts.setdefault(name, set()).add(int(count) if count.isdigit() else _kernel_constant(count))
    assert all(len(c) == 1 for c in counts.values()), counts
    return {name: c.pop() for name, c in counts.items()}


def pass_at(j, N):                                   # render_fused_ws3.cu: pass_at
    if j == 0:
        return (0, 0)
    if N == 1:
        return (0, 1)
    if j == 1:
        return (1, 0)
    k, body = j - 2, 2 * (N - 2)
    if k < body:
        return ((k >> 1) + 2, 0) if (k & 1) else (k >> 1, 1)
    return (N - 2 + (k - body), 1)


def tile_at(q, N):
    j = q // 3
    n, p = pass_at(j, N)
    return (n, p, q - 3 * j)


class Bar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def passed(self, parity):                        # mbarrier.try_wait.parity
        return (self.phase & 1) != parity


class TxBar(Bar):                                    # mbarrier with a transaction count (arrive.expect_tx / complete_tx)
    def __init__(self, count):
        super().__init__(count)
        self.tx = 0

    def _flip(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive_expect_tx(self):
        self.tx += 1
        self.pending -= 1
        assert self.pending >= 0
        self._flip()

    def complete_tx(self):
        self.tx -= 1
        assert self.tx >= 0
        self._flip()


class Sim:
    def __init__(self, N, seed, S=96, sig_count=ARRIVALS['sigc_ready'], stored_wait='all', staging_wait=True,
                 col_stored_wait=True, coarse_guard=True, fine_guard=True, fine_areas=2, reload_after_read=True):
        # The kernel's choices; the other values model bugs that the negative controls below must catch:
        #   sig_count          arrivals of sigc_ready / sigf_ready (every decoder warp)
        #   stored_wait        the bulk wait before arriving on col_stored: 'all' (wait_group 0) | 'read' (wait_group.read 0)
        #   staging_wait       the .read wait before a warpgroup rewrites its staging tile
        #   col_stored_wait    the ray warps wait on col_stored before their first loads of a group
        #   coarse_guard       the decoder waits for state_free of group m - 3 before its first store into CA[m % 3]
        #   fine_guard         ... of group m - 2 before its first store into FA[m % fine_areas]
        #   fine_areas         fine colour areas (2: FA[n & 1])
        #   reload_after_read  a ray warp reloads a buffer after reading it (else right after its col_full wait)
        self.N, self.T, self.S, self.rng = N, 6 * N, S, random.Random(seed)
        self.stored_wait, self.staging_wait, self.col_stored_wait = stored_wait, staging_wait, col_stored_wait
        self.coarse_guard, self.fine_guard, self.fine_areas = coarse_guard, fine_guard, fine_areas
        self.reload_after_read = reload_after_read
        A = ARRIVALS
        self.a1_full = [Bar(A['a1_full']) for _ in range(K_NA)]; self.a1_empty = [Bar(A['a1_empty']) for _ in range(K_NA)]
        self.fine_ready = [Bar(A['fine_ready']) for _ in range(K_STATES)]
        self.state_free = [Bar(A['state_free']) for _ in range(K_STATES)]
        self.sigc_ready = [Bar(sig_count) for _ in range(K_STATES)]; self.sigf_ready = [Bar(sig_count) for _ in range(K_STATES)]
        self.col_stored = [Bar(A['col_stored']) for _ in range(2)]
        self.col_full = [[TxBar(A['col_full']) for _ in range(K_COL_BUFS)] for _ in range(K_RW)]
        self.now, self.events, self.seq = 0.0, [], 0
        # hazard bookkeeping
        self.a1_tile, self.a1_written, self.a1_read = [None] * K_NA, [0] * K_NA, [0] * K_NA
        self.sigma_writes = {}                        # (group, pass) -> decoder warp-tiles that stored their sigma rows
        self.importance_done, self.colours_done = set(), set()
        self.colours_warps = {}                       # group -> ray warps that finished its colours
        self.state_owner = [None] * K_STATES
        self.bulk_groups = [[], []]                   # per warpgroup: its elected thread's bulk-store groups
        self.col_signalled = set()                    # groups whose col_stored phase completed
        self.area_content = {}                        # (area, block) -> (group, tile) whose store completed there
        self.area_last = {}                           # (area, block) -> (group, tile) last stored there
        self.load_done = set()                        # (group, tile, block) whose load landed
        self.buf = [[None] * K_COL_BUFS for _ in range(K_RW)]          # [warp][b] -> (group, tile, landed?)
        self.buf_read = [[False] * K_COL_BUFS for _ in range(K_RW)]
        self.wg_count, self.wg_gen = [0, 0], [0, 0]

    def dur(self, lo, hi):
        return self.rng.uniform(lo, hi)

    def later(self, dt, fn):
        self.seq += 1
        heapq.heappush(self.events, (self.now + dt, self.seq, fn))

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
        # Each delay of a bulk copy is usually short and now and then (a busy SM or a congested L2) much longer than a tile,
        # so that every hazard check can fire when the wait that guards it is missing.
        t_read = self.dur(0.05, 1.0) if self.rng.random() < 0.9 else self.dur(1.0, 20.0)
        self.later(t_read, lambda: rec.__setitem__('read', True))

        def written():
            rec['all'] = True
            for blk in range(4 * h, 4 * h + 4):
                self.area_content[(area, blk)] = (n, 3 * p + k)
        self.later(t_read + (self.dur(0.05, 4.0) if self.rng.random() < 0.9 else self.dur(4.0, 40.0)), written)

    def bulk_wait(self, h, kind):                    # cp.async.bulk.wait_group{.read} 0
        yield ('until', lambda: all(r[kind] for r in self.bulk_groups[h]))
        if kind == 'all':
            self.bulk_groups[h] = []

    def ray_load(self, rw, n, t):                    # lane 0 of ray warp rw: its blocks of tile t into col_buf[t % kColBufs]
        p, k = divmod(t, 3)
        b, area = t % K_COL_BUFS, self.area(n, p, k)
        blocks = self.blocks(rw)
        assert n in self.col_signalled, f'load of {area} for group {n} (warp {rw}) issued before col_stored signalled the group'
        assert all(self.area_content.get((area, blk)) == (n, t) for blk in blocks), \
            f'load of {area} for group {n} (warp {rw}) issued before the bulk stores of its rows completed'
        assert self.buf[rw][b] is None or self.buf_read[rw][b], f'col_buf[{b}] rows of warp {rw} reloaded before it read them'
        self.col_full[rw][b].arrive_expect_tx()
        self.buf[rw][b], self.buf_read[rw][b] = (n, t, False), False

        def landed():
            self.buf[rw][b] = (n, t, True)
            for blk in blocks:
                self.load_done.add((n, t, blk))
            self.col_full[rw][b].complete_tx()
        self.later(self.dur(0.2, 3.0) if self.rng.random() < 0.9 else self.dur(3.0, 30.0), landed)

    # ---------------------------------------------------------------- roles (generators yield ('wait', bar, parity) |
    # ('until', predicate) | ('work', dt) | ('wgbar', warpgroup))
    def gather_warp(self, gw):
        team, it = gw // (K_GW // K_TEAMS), 0
        for q in range(self.T):
            n, p, k = tile_at(q, self.N)
            my_it = it; it += 1
            if my_it % K_TEAMS != team:
                continue
            si, par = n % K_STATES, (n // K_STATES) & 1
            if p == 0:
                yield ('wait', self.state_free[si], par ^ 1)
                prev = self.state_owner[si]
                assert prev is None or prev == n or prev in self.colours_done, f'state slot of group {prev} rewritten for {n}'
                self.state_owner[si] = n
            else:
                yield ('wait', self.fine_ready[si], par)
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
        mark = {'stored': -1, 'signalled': -1}       # last group whose fine pass was stored / signalled

        def signal_stored():
            if elect:
                yield from self.bulk_wait(h, self.stored_wait)
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
            assert self.a1_tile[stage] == it and self.a1_written[stage] == ARRIVALS['a1_full'], \
                f'decoder reads A1 stage {stage} before tile {it} is complete'
            yield ('work', self.dur(0.5, 2))          # layer 1 (wgmma from shared memory)
            self.a1_read[stage] += 1
            self.a1_empty[stage].arrive()
            yield ('work', self.dur(1, 4))            # softplus, layer 2 from registers
            if mark['stored'] > mark['signalled']:
                yield from signal_stored()
            elif elect and self.staging_wait:
                yield from self.bulk_wait(h, 'read')
            yield ('wgbar', h)
            assert all(r['read'] for r in self.bulk_groups[h]), f'staging of warpgroup {h} rewritten before its bulk store read it'
            yield ('work', self.dur(0.2, 1))          # staging and sigma stores
            self.sigma_writes[(n, p)] = self.sigma_writes.get((n, p), 0) + 1
            yield ('wgbar', h)
            if elect:
                prev = n - (3 if p == 0 else 2)
                if k == 0 and prev >= 0 and (self.coarse_guard if p == 0 else self.fine_guard):
                    yield ('wait', self.state_free[prev % K_STATES], (prev // K_STATES) & 1)
                self.bulk_store(h, n, p, k)
            if k == 2:
                if p == 1:
                    mark['stored'] = n
                (self.sigc_ready if p == 0 else self.sigf_ready)[n % K_STATES].arrive()
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
                yield ('work', self.dur(2, 12))       # composite: omega / pos of the warp's own rays
                yield from self.colours(rw, n)
                self.colours_warps[n] = self.colours_warps.get(n, 0) + 1
                if self.colours_warps[n] == K_RW:
                    self.colours_done.add(n)
                self.state_free[si].arrive()

    def procs(self):
        return ([('G%d' % g, self.gather_warp(g)) for g in range(K_GW)] + [('E%d' % e, self.decoder_warp(e)) for e in range(K_EW)] +
                [('R%d' % r, self.ray_warp(r)) for r in range(K_RW)])

    # ---------------------------------------------------------------- scheduler
    def run(self):
        procs = self.procs()
        state = {name: ('ready', None) for name, _ in procs}          # ready | wait | until | sleep | wgbar | done
        gens = dict(procs)

        def step(name):
            try:
                op = next(gens[name])
            except StopIteration:
                state[name] = ('done', None)
                return
            if op[0] in ('wait', 'until'):
                state[name] = (op[0], op[1:])
            elif op[0] == 'work':
                state[name] = ('sleep', None)
                self.later(op[1], lambda name=name: state.__setitem__(name, ('ready', None)))
            else:                                    # bar.sync of the warpgroup's four warps
                h = op[1]
                self.wg_count[h] += 1
                state[name] = ('wgbar', (h, self.wg_gen[h]))
                if self.wg_count[h] == 4:
                    self.wg_count[h] = 0
                    self.wg_gen[h] += 1

        def runnable(st, arg):
            return (st == 'ready' or (st == 'wait' and arg[0].passed(arg[1])) or (st == 'until' and arg[0]())
                    or (st == 'wgbar' and arg[1] != self.wg_gen[arg[0]]))
        guard = 0
        while True:
            guard += 1
            assert guard < 5_000_000
            ready = [name for name, (st, arg) in state.items() if runnable(st, arg)]
            if ready:
                step(self.rng.choice(ready))
                continue
            if self.events:
                t, _, fn = heapq.heappop(self.events)
                self.now = t
                fn()
                continue
            break
        stuck = {n: s for n, s in state.items() if s[0] != 'done'}
        assert not stuck, f'deadlock with N={self.N}: {sorted(stuck)[:6]}'
        assert self.colours_done == set(range(self.N))


def test_pass_schedule_visits_every_group_once_in_a_valid_order():
    for N in range(1, 12):
        seq = [pass_at(j, N) for j in range(2 * N)]
        assert sorted(seq) == sorted([(n, p) for n in range(N) for p in (0, 1)])
        pos = {np_: i for i, np_ in enumerate(seq)}
        for n in range(N):
            assert pos[(n, 0)] < pos[(n, 1)]                                       # F(n) after C(n)
            if n + 1 < N:
                assert pos[(n, 1)] < pos[(n + 1, 1)] and pos[(n, 0)] < pos[(n + 1, 0)]
            if n + 3 < N:
                assert pos[(n + 1, 1)] < pos[(n + 3, 0)]                           # CA[n % 3] is free again before C(n+3)
            if N > 2 and 1 <= n and n + 1 < N:
                assert pos[(n + 1, 0)] < pos[(n, 1)]                               # >= one pass of slack for importance(n)


def test_model_sizes_and_arrival_counts_are_the_kernels():
    assert (K_GW, K_EW, K_RW, K_TEAMS, K_NA, K_STATES, K_COL_BUFS) == (12, 8, 4, 3, 3, 4, 2)
    assert 6 % K_COL_BUFS == 0          # colours() walks a group's six tiles through the buffers in whole rounds
    assert _mbar_init_counts() == ARRIVALS


@pytest.mark.parametrize('S', [96, 48])
@pytest.mark.parametrize('N', [1, 2, 3, 4, 5, 7, 8, 13])
def test_protocol_has_no_deadlock_or_hazard(N, S):
    # 24 distinct seeds (the two progressions share s = 0)
    for seed in [s * 101 + N for s in range(12)] + [s * 131 + N for s in range(1, 13)]:
        Sim(N, seed, S=S).run()


@pytest.mark.parametrize('kw, match', [
    # with four of the eight decoder warps counted on sigc_ready / sigf_ready, the ray warps start on sigma not all stored
    pytest.param(dict(sig_count=4), r'before every (coarse|fine) sigma was stored', id='short_sigma_hand_off'),
    # with only a .read wait before col_stored (the staging tile is free, the global writes may still be in flight), a ray
    # warp loads colours whose stores have not completed
    pytest.param(dict(stored_wait='read'), 'issued before the bulk stores of its rows completed', id='read_wait_before_col_stored'),
    # without the .read wait before the epilogue, a warpgroup rewrites its staging tile while the previous tile's bulk store
    # may still be reading it
    pytest.param(dict(staging_wait=False), 'rewritten before its bulk store read it', id='no_staging_wait'),
    # without the col_stored wait, a ray warp loads colours before the decoder signalled them
    pytest.param(dict(col_stored_wait=False), 'issued before col_stored signalled the group', id='no_col_stored_wait'),
    # without the coarse area's guard, C(m) overwrites CA[m % 3] while group m - 3's loads may be in flight
    pytest.param(dict(coarse_guard=False), r'coarse area .* overwritten before its load landed', id='no_coarse_guard'),
    # a reload issued right after the col_full wait overwrites rows the warp has not read
    pytest.param(dict(reload_after_read=False), 'reloaded before it read them', id='reload_before_read'),
    # with a single fine area and no guard, F(m + 1) overwrites it while group m's loads may be in flight
    pytest.param(dict(fine_areas=1, fine_guard=False), r"fine area \('FA', 0, \d\) .* overwritten before its load landed", id='one_fine_area_unguarded'),
])
@pytest.mark.parametrize('S', [96, 48])
def test_simulation_catches_each_protocol_bug(kw, match, S):
    # the coarse areas have about five tiles of slack, so their hazard needs a long bulk-copy tail: up to 200 seeds
    with pytest.raises(AssertionError, match=match):
        for seed in range(200):
            Sim(13, seed, S=S, **kw).run()
