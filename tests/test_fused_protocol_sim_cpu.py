"""CPU: discrete-event simulation of the mbarrier and bulk-copy protocol of the fused renderer (csrc/render_fused_ws3.cu):
its pass schedule and the hand-off between its 24 warps - 12 gather, 8 decoder (two wgmma warpgroups), 4 ray.  Every role's
control flow is transcribed from the CUDA source (same loops, same barriers, parities and arrival counts, the same
placement of colours(n) and its named barriers, the elected threads' bulk groups with their .read and full waits); work
items get random durations and the runnable warps are stepped in random order, over many seeds and group counts.  Bulk
copies run asynchronously with random read / write / landing delays, each with a tail longer than a tile, so that a check
fires whenever the wait guarding it is missing (the negative controls at the end).  Asserted:
  * no deadlock and no lost mbarrier phase (a waiter that a barrier overtakes by two phases blocks forever), and every
    group's colours run once;
  * A1 ring: the gather rewrites a stage only after all eight decoder warps have read its previous tile, and a decoder warp
    reads a stage only once all four warps of the team have written it;
  * shared-memory hazards: the ray warps read a pass's sigma only after every decoder warp wrote its rows, a per-group state
    slot is not rewritten by the gather before its previous group is finished, the omega slot not before its previous
    group's colours are done, fine depths are read only after importance;
  * colour path: a warpgroup's staging tile is not rewritten before its last bulk store has read it; no load of a colour
    area half is issued before the store that wrote it completed; colours(n) reads a col_buf half only after its load
    landed (complete_tx), and a load does not overwrite a half that colours() is still reading; CA[n % 3] and FA are not
    rewritten before the loads of their previous group completed.
It mirrors the protocol, not the arithmetic; parity on hardware is what tests/test_render_gpu.py is for."""
import heapq
import random

import pytest

K_NA, K_EW, K_RW, K_TEAMS = 4, 8, 4, 3
K_COL_BUFS = 3                                       # kColBufs


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
    def __init__(self, N, seed, sig_count=K_EW, first_wait='all', staging_wait=True, colours_k=0):
        # The kernel's choices; the other values model bugs that the negative controls below must catch:
        #   sig_count     arrivals of sigc_ready / sigf_ready (every decoder warp, K_EW)
        #   first_wait    the bulk wait before a group's first loads: 'all' (wait_group 0) | 'read' (wait_group.read 0)
        #   staging_wait  the .read wait before a warpgroup rewrites its staging tile
        #   colours_k     colours(n) runs at the top of tile colours_k of F(n+1) (0: before F(n+1) stores to FA)
        self.N, self.T, self.rng = N, 6 * N, random.Random(seed)
        self.first_wait, self.staging_wait, self.colours_k = first_wait, staging_wait, colours_k
        B = Bar
        self.a1_full = [B(4) for _ in range(K_NA)]; self.a1_empty = [B(K_EW) for _ in range(K_NA)]
        self.fine_ready = [B(K_RW) for _ in range(4)]; self.state_free = [B(1) for _ in range(4)]
        self.sigc_ready = [B(sig_count) for _ in range(4)]; self.sigf_ready = [B(sig_count) for _ in range(4)]
        self.omega_ready = [B(K_RW) for _ in range(2)]
        self.col_full = [TxBar(2) for _ in range(K_COL_BUFS)]
        self.now, self.events, self.seq = 0.0, [], 0
        # hazard bookkeeping
        self.a1_tile, self.a1_written, self.a1_read = [None] * K_NA, [0] * K_NA, [0] * K_NA
        self.sigma_writes = {}                        # (group, pass) -> decoder warp-tiles that stored their sigma rows
        self.colours_done, self.importance_done, self.composite_done = set(), set(), set()
        self.state_owner = [None] * 4
        self.slot_owner = [None] * 2
        self.bulk_groups = [[], []]                   # per warpgroup: its elected thread's bulk-store groups
        self.area_content = {}                        # (area, half) -> (group, pass, k) whose store completed there
        self.area_last = {}                           # (area, half) -> (group, pass, k) last stored there
        self.load_done = set()                        # (group, t, half) whose load landed
        self.buf = [[None, None] for _ in range(K_COL_BUFS)]      # [b][half] -> (group, t, landed?)
        self.buf_reads = [[0, 0] for _ in range(K_COL_BUFS)]
        self.ebar_count, self.ebar_gen = 0, 0
        self.wg_count, self.wg_gen = [0, 0], [0, 0]

    def dur(self, lo, hi):
        return self.rng.uniform(lo, hi)

    def later(self, dt, fn):
        self.seq += 1
        heapq.heappush(self.events, (self.now + dt, self.seq, fn))

    @staticmethod
    def area(n, p, k):
        return ('CA', n % 3, k) if p == 0 else ('FA', k)

    # ---------------------------------------------------------------- bulk copies of the elected thread of warpgroup h
    def bulk_store(self, h, n, p, k):
        key = (self.area(n, p, k), h)
        prev = self.area_last.get(key)
        if prev is not None:
            m, pp, kk = prev
            assert (m, 3 * pp + kk, h) in self.load_done, f'{key} of group {m} overwritten before its load completed'
        self.area_last[key] = (n, p, k)
        rec = {'read': False, 'all': False}
        self.bulk_groups[h].append(rec)
        # Each delay of a bulk copy is usually short and now and then (a busy SM or a congested L2) much longer than a tile,
        # so that every hazard check below can fire when the wait that guards it is missing.
        t_read = self.dur(0.05, 1.0) if self.rng.random() < 0.9 else self.dur(1.0, 20.0)
        self.later(t_read, lambda: rec.__setitem__('read', True))

        def written():
            rec['all'] = True
            self.area_content[key] = (n, p, k)
        self.later(t_read + (self.dur(0.05, 4.0) if self.rng.random() < 0.9 else self.dur(4.0, 40.0)), written)

    def bulk_wait(self, h, kind):                    # cp.async.bulk.wait_group{.read} 0
        yield ('until', lambda: all(r[kind] for r in self.bulk_groups[h]))
        if kind == 'all':
            self.bulk_groups[h] = []

    def bulk_load(self, h, n, t):
        p, k = divmod(t, 3)
        b, key = t % K_COL_BUFS, (self.area(n, p, k), h)
        assert self.area_content.get(key) == (n, p, k), f'load of {key} for group {n} issued before its store completed'
        assert self.buf[b][h] is None or self.buf_reads[b][h] == 4, f'col_buf[{b}] half {h} reloaded while colours() reads it'
        self.col_full[b].arrive_expect_tx()
        self.buf[b][h], self.buf_reads[b][h] = (n, t, False), 0

        def landed():
            self.buf[b][h] = (n, t, True)
            self.load_done.add((n, t, h))
            self.col_full[b].complete_tx()
        self.later(self.dur(0.2, 3.0) if self.rng.random() < 0.9 else self.dur(3.0, 30.0), landed)

    # ---------------------------------------------------------------- roles (generators yield ('wait', bar, parity) |
    # ('until', predicate) | ('work', dt) | ('ebar',) | ('wgbar', warpgroup))
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
        mark = {'stored': -1, 'loaded': -1}

        def first_loads(n):
            if elect:
                yield from self.bulk_wait(h, self.first_wait)
                for t in range(K_COL_BUFS):
                    self.bulk_load(h, n, t)
            mark['loaded'] = n

        def colours(n):
            if mark['loaded'] < n:
                yield from first_loads(n)
            yield ('wait', self.omega_ready[n & 1], (n >> 1) & 1)
            assert n in self.composite_done and self.slot_owner[n & 1] == n
            for t in range(6):
                b = t % K_COL_BUFS
                yield ('wait', self.col_full[b], ((6 * n + t) // K_COL_BUFS) & 1)
                assert self.buf[b][h] == (n, t, True), f'colours({n}) reads col_buf[{b}] before tile {t} landed'
                yield ('work', self.dur(0.2, 1.5))
                assert self.buf[b][h] == (n, t, True), f'col_buf[{b}] changed while colours({n}) read it'
                self.buf_reads[b][h] += 1
                if t + K_COL_BUFS < 6:
                    yield ('wgbar', h)
                    if elect:
                        self.bulk_load(h, n, t + K_COL_BUFS)
            yield ('ebar',)
            yield ('work', self.dur(0.1, 0.5))
            yield ('ebar',)
            if e == 0:
                self.colours_done.add(n)
                self.state_free[n & 3].arrive()

        for it in range(self.T):
            n, p, k = tile_at(it, self.N)
            if p == 1 and k == self.colours_k and n >= 1:
                yield from colours(n - 1)
            stage = it % K_NA
            yield ('wait', self.a1_full[stage], (it // K_NA) & 1)
            assert self.a1_tile[stage] == it and self.a1_written[stage] == 4, f'decoder reads A1 stage {stage} before tile {it} is complete'
            yield ('work', self.dur(0.5, 2))          # layer 1 (wgmma from shared memory)
            self.a1_read[stage] += 1
            self.a1_empty[stage].arrive()
            yield ('work', self.dur(1, 4))            # softplus, layer 2 from registers
            if mark['stored'] > mark['loaded']:
                yield from first_loads(mark['stored'])
            elif elect and self.staging_wait:
                yield from self.bulk_wait(h, 'read')
            yield ('wgbar', h)
            assert all(r['read'] for r in self.bulk_groups[h]), f'staging of warpgroup {h} rewritten before its bulk store read it'
            yield ('work', self.dur(0.2, 1))          # staging and sigma stores
            self.sigma_writes[(n, p)] = self.sigma_writes.get((n, p), 0) + 1
            yield ('wgbar', h)
            if elect:
                self.bulk_store(h, n, p, k)
            if k == 2:
                if p == 1:
                    mark['stored'] = n
                (self.sigc_ready if p == 0 else self.sigf_ready)[n & 3].arrive()
        yield from colours(self.N - 1)

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
                if n >= 2:
                    yield ('wait', self.state_free[(n - 2) & 3], ((n - 2) >> 2) & 1)
                    assert (n - 2) in self.colours_done
                prev = self.slot_owner[n & 1]
                assert prev is None or prev == n or prev in self.colours_done, f'omega slot of group {prev} rewritten for {n}'
                self.slot_owner[n & 1] = n
                yield ('work', self.dur(2, 12))
                if rw == 0:
                    self.composite_done.add(n)
                self.omega_ready[n & 1].arrive()

    def procs(self):
        return ([('G%d' % g, self.gather_warp(g)) for g in range(12)] + [('E%d' % e, self.decoder_warp(e)) for e in range(K_EW)] +
                [('R%d' % r, self.ray_warp(r)) for r in range(K_RW)])

    # ---------------------------------------------------------------- scheduler
    def run(self):
        procs = self.procs()
        state = {name: ('ready', None) for name, _ in procs}          # ready | wait | until | sleep | ebar | wgbar | done
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
            elif op[0] == 'wgbar':
                h = op[1]
                self.wg_count[h] += 1
                state[name] = ('wgbar', (h, self.wg_gen[h]))
                if self.wg_count[h] == 4:
                    self.wg_count[h] = 0
                    self.wg_gen[h] += 1
            else:
                self.ebar_count += 1
                state[name] = ('ebar', self.ebar_gen)
                if self.ebar_count == K_EW:
                    self.ebar_count = 0
                    self.ebar_gen += 1

        def runnable(st, arg):
            return (st == 'ready' or (st == 'wait' and arg[0].passed(arg[1])) or (st == 'until' and arg[0]())
                    or (st == 'ebar' and arg != self.ebar_gen) or (st == 'wgbar' and arg[1] != self.wg_gen[arg[0]]))
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


@pytest.mark.parametrize('N', [1, 2, 3, 4, 5, 7, 8, 13])
def test_protocol_has_no_deadlock_or_hazard(N):
    # 24 distinct seeds (the two progressions share s = 0)
    for seed in [s * 101 + N for s in range(12)] + [s * 131 + N for s in range(1, 13)]:
        Sim(N, seed).run()


def test_simulation_catches_a_short_sigma_hand_off():
    """The model is not vacuous: with half the decoder warps counted on sigc_ready / sigf_ready (the arrival count of the
    earlier design, where four warps read sigma back) the ray warps start on sigma that is not all stored yet."""
    with pytest.raises(AssertionError, match='sigma was stored'):
        for seed in range(40):
            Sim(4, seed, sig_count=4).run()


def test_simulation_catches_a_read_only_wait_before_the_loads():
    """With only a .read wait (the staging tile is free, the global writes may still be in flight) before a group's first
    loads, a load starts on a colour area half that is not written yet."""
    with pytest.raises(AssertionError, match='issued before its store completed'):
        for seed in range(40):
            Sim(4, seed, first_wait='read').run()


def test_simulation_catches_a_missing_staging_wait():
    """Without the .read wait before the epilogue, a warpgroup rewrites its staging tile while the bulk store of the
    previous tile may still be reading it."""
    with pytest.raises(AssertionError, match='rewritten before its bulk store read it'):
        for seed in range(40):
            Sim(4, seed, staging_wait=False).run()


def test_simulation_catches_colours_after_the_fine_area_is_rewritten():
    """With colours(n) one tile later (at the top of F(n+1)'s second tile), F(n+1)'s first tile is stored to the fine area
    before colours(n) has loaded group n's copy of it."""
    with pytest.raises(AssertionError, match='overwritten before its load completed'):
        for seed in range(40):
            Sim(4, seed, colours_k=1).run()
