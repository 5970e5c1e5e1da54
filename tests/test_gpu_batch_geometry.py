"""GPU: every batched State kernel of every rule-core instantiation at the batch sizes it runs at, against the oracle.

The lock-step tests pin the rule logic at batches of at most one block.  What depends on the batch geometry — the ILP slots
past lane 256, a warp that holds fewer than 32 live lanes (the warp-staged mask store, the observation tile), the chunk
offsets of the host-buffer step, the lane clones and the error record — is checked here:

- Per game, a pool of K oracle states from seeded random play (initial state, chance nodes, terminal states and depths in
  between), driven through a K-lane device batch, with tables of every observable of each pool state and of three children.
- A batch of capacity n + 40 is filled by b2s_gather_states, lane i holding pool state perm[i], so every expected value is a
  table lookup; n runs over 1, 31, 33, 256 ILP - 1, 256 ILP + 1 and 3 * 256 ILP + 17 (ILP = lanes per thread of the rule
  core).  Lanes [n, n + 40) must come out of every call unchanged, and every output has a sentinel-filled guard of 32 rows on
  either side that must stay intact.
- Read kernels (status, legal masks, legal lists, observation and information-state tensors) and every stepping entry point
  (apply_actions, the fused step, the host-buffer steps on their stream, graph, zero-copy and chunked paths) with skipped,
  legal, illegal and terminal-lane actions: rejected lanes keep their state and are counted, and the lowest is reported.
- Clones (copy, broadcast, gather) of mid-game go and breakthrough lanes, history column included."""
import ctypes as C
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import open_spiel_b200 as b2
from open_spiel_b200 import _lib
from oracle_lib import OracleGame

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

# game string -> lanes per thread of its rule core (kIlp)
GAMES = {
    "tic_tac_toe": 4,
    "connect_four": 4,                         # compile-time 6x7 core
    "connect_four(rows=5,columns=6)": 4,       # general core
    "breakthrough": 2,                         # 24 mask words
    "hex(board_size=5)": 1,
    "hex(board_size=4,swap=True)": 1,
    "go(board_size=9)": 1,                     # 128-bit core, history column
    "go(board_size=13)": 1,                    # 384-bit core, 12 mask words
    "kuhn_poker": 4,
    "kuhn_poker(players=3)": 4,
    "leduc_poker": 4,
    "leduc_poker(players=4)": 2,               # 4 players
    "mnk": 1,
    "othello": 2,
    "y(board_size=9)": 1,
    "havannah(board_size=4,swap=True)": 1,
}
K = 240            # pool states per game
G = 32             # guard rows on either side of every output
TAIL = 40          # lanes past n that every call must leave alone
SENT32 = 0x7FBADBAD          # int32 / float32 (a NaN) guard pattern
SENT16 = -7222
SENT8 = 0xA5


def sizes(ilp):
    t = 256 * ilp
    return [1, 31, 33, t - 1, t + 1, 3 * t + 17]


# ---- pool and tables ---------------------------------------------------------------------------------------------------------

class Pool:
    """K oracle states and a K-lane device batch holding the same states; tables of the observables of node 4k (pool state k)
    and 4k + 1..3 (its children by actions act[k, 0..2]: first, last and a random legal action; the state itself when
    terminal).  bad[k] = the lowest action id that is not legal in state k, -1 if every id is legal."""

    def __init__(self, gs, seed):
        self.gs = gs
        self.game, og = b2.load_game(gs), OracleGame(gs)
        info = self.game._info
        self.P, self.W, self.A = info.num_players, info.mask_words, info.num_distinct_actions
        self.width = max(self.A, info.max_chance_outcomes)
        self.F, self.I = info.observation_tensor_size, info.information_state_tensor_size
        self.batch = self.game.new_batch(K)
        rng = np.random.RandomState(seed)
        states = [og.new_initial_state() for _ in range(K)]
        L = og.max_game_length
        depth = rng.randint(0, min(L, 120) + 1, size=K)
        depth[0] = 0                                  # the initial state
        depth[1::8] = 10 ** 6                         # played to the end
        ply = 0
        while True:
            acts = np.full(K, -1, dtype=np.int32)
            for i, st in enumerate(states):
                if ply < depth[i] and not st.is_terminal():
                    la = st.legal_actions()
                    acts[i] = la[rng.randint(len(la))]
                    st.apply_action(int(acts[i]))
            if (acts == -1).all():
                break
            self.batch.apply_actions(torch.from_numpy(acts).cuda())
            ply += 1
        assert self.batch.error_count()[0] == 0
        nodes, self.act = [], np.zeros((K, 3), dtype=np.int64)
        self.bad = np.full(K, -1, dtype=np.int64)
        for k, st in enumerate(states):
            nodes.append(st)
            la = st.legal_actions()
            if st.is_terminal():
                nodes += [st, st, st]
                continue
            missing = sorted(set(range(self.width)) - set(la))
            self.bad[k] = missing[0] if missing else -1
            for j, a in enumerate((la[0], la[-1], la[rng.randint(len(la))])):
                self.act[k, j] = a
                c = st.clone()
                c.apply_action(a)
                nodes.append(c)
        N = len(nodes)
        self.cur = np.array([s.current_player() for s in nodes], dtype=np.int64)
        self.term = np.array([s.is_terminal() for s in nodes], dtype=np.uint8)
        self.rets = np.array([s.returns() for s in nodes], dtype=np.float32).view(np.int32)
        self.legal = np.full((N, self.width), SENT16, dtype=np.int16)
        self.count = np.zeros(N, dtype=np.int32)
        words = np.zeros((N, self.W), dtype=np.uint64)
        for j, s in enumerate(nodes):
            la = s.legal_actions()
            self.count[j] = len(la)
            self.legal[j, :len(la)] = la
            for a in la:
                words[j, a // 32] |= 1 << (a % 32)
        self.words = words.astype(np.uint32).view(np.int32)
        self.obs = np.stack([np.stack([s.observation_tensor(p) for p in range(self.P)]) for s in nodes])
        self.info = (np.stack([np.stack([s.information_state_tensor(p) for p in range(self.P)]) for s in nodes])
                     if self.I else None)
        self.terminal_pool = self.term[0::4].astype(bool)
        # status byte of b2s_step_fused_host_compact
        r0 = self.rets.view(np.float32)[:, 0]
        small = self.A <= 7
        self.status = np.where(self.term == 1, 0x80 | np.where(r0 > 0, 1, np.where(r0 < 0, 2, 0)),
                               (self.words[:, 0] & 0x7F) if small else 0).astype(np.uint8)

    def fill(self, perm, batch=None):
        """A batch (new, of capacity len(perm), or `batch`) whose lane i holds pool state perm[i], by b2s_gather_states."""
        b = batch if batch is not None else self.game.new_batch(len(perm))
        idx = torch.from_numpy(np.ascontiguousarray(perm, dtype=np.int64)).cuda()
        _lib.check(_lib.lib().b2s_gather_states(b._h, self.batch._h, C.c_void_p(idx.data_ptr()), len(perm), b._stream()))
        torch.cuda.synchronize()
        b._reset_errors()
        return b

    def wld(self):
        """b2s_step_fused_host_compact serves win / loss / draw games without chance nodes."""
        info = self.game._info
        return info.min_utility == -1.0 and info.max_utility == 1.0 and info.max_chance_outcomes == 0

    def actions(self, perm, n, seed, illegal=True, terminal=True):
        """Per lane i < n an action and the node it leads to: -1 (skip), a child action, an illegal id or any action on a
        terminal lane (both rejected: the lane keeps its state).  Returns (actions [len(perm)] int32, expected node [n],
        rejected lanes).  Lanes >= n get their first child's action, so a kernel that steps past n would change them."""
        rng = np.random.RandomState(seed)
        k = perm[:n]
        cat = rng.randint(0, 5, size=n)
        acts = np.full(len(perm), -1, dtype=np.int64)
        node = 4 * k.copy()
        term = self.terminal_pool[k]
        child = (cat >= 1) & (cat <= 3) & ~term
        acts[:n][child] = self.act[k[child], cat[child] - 1]
        node[child] += cat[child]
        bad = (cat == 4) & ~term & (self.bad[k] >= 0) if illegal else np.zeros(n, bool)
        acts[:n][bad] = self.bad[k[bad]]
        on_term = (cat >= 1) & term if terminal else np.zeros(n, bool)
        acts[:n][on_term] = self.act[k[on_term], 0]            # 0: any action id
        tail = perm[n:]
        acts[n:] = np.where(self.terminal_pool[tail], -1, self.act[tail, 0])
        return acts.astype(np.int32), node, np.nonzero(bad | on_term)[0]


@functools.lru_cache(maxsize=None)
def pool_of(gs):
    return Pool(gs, seed=sum(map(ord, gs)) % 1000)


def perm_for(n, seed):
    return np.random.RandomState(seed).randint(0, K, size=n + TAIL).astype(np.int64)


# ---- guarded buffers ---------------------------------------------------------------------------------------------------------

class Guarded:
    """rows x width elements of `dtype` with G sentinel rows before and after (plus `offset` extra leading elements): .ptr is
    row 0 of the payload, .rows() the payload, .intact() whether the guards still hold the sentinel."""

    def __init__(self, rows, width, dtype, sentinel, offset=0, device="cuda", pin=False):
        self.rows_, self.width, self.lead = rows, width, G * width + offset
        self.t = torch.full((self.lead + (rows + G) * width,), sentinel, dtype=dtype, device=device)
        if pin:
            self.t = self.t.pin_memory()
        self.sentinel = sentinel
        self.ptr = self.t.data_ptr() + self.lead * self.t.element_size()

    def view(self):
        return self.t[self.lead:self.lead + self.rows_ * self.width]

    def rows(self):
        return self.view().cpu().numpy().reshape(self.rows_, self.width)

    def intact(self):
        a = self.t.cpu().numpy()
        return bool((a[:self.lead] == self.sentinel).all() and (a[self.lead + self.rows_ * self.width:] == self.sentinel).all())


def out32(rows, width, offset=0):
    return Guarded(rows, width, torch.int32, SENT32, offset)


def tail_blobs(batch, n):
    return [batch.state_blob(i) for i in range(n, batch.n)]


def lane_key(batch, lane):
    """A lane's blob with go's history column cut after the entries the state uses (hashes 0..ply; the rest is scratch)."""
    b = batch.state_blob(lane)
    info = batch.info
    if info.history_bytes:
        sb = info.state_bytes
        ply = (int.from_bytes(b[12:16], "little") >> 11) & 1023 if sb == 32 else (int.from_bytes(b[96:104], "little") >> 13) & 1023
        b = b[:sb + 8 * (ply + 1)]
    return b


def observe(pool, batch, n):
    """status, legal mask words and every player's observation of lanes [0, n), through the plain entry points."""
    cur, term, rets = (t.cpu().numpy() for t in batch.status(n=n))
    return {"cur": cur.astype(np.int64), "term": term, "rets": rets.view(np.int32),
            "words": batch.legal_actions_mask_words(n=n).cpu().numpy(),
            "obs": [batch.observation_tensor(p, n=n).cpu().numpy() for p in range(pool.P)]}


def assert_state(pool, batch, n, node, what):
    o = observe(pool, batch, n)
    np.testing.assert_array_equal(o["cur"], pool.cur[node], err_msg=what)
    np.testing.assert_array_equal(o["term"], pool.term[node], err_msg=what)
    np.testing.assert_array_equal(o["rets"], pool.rets[node], err_msg=what)
    np.testing.assert_array_equal(o["words"], pool.words[node], err_msg=what)
    for p in range(pool.P):
        np.testing.assert_array_equal(o["obs"][p], pool.obs[node, p], err_msg="%s obs %d" % (what, p))
    return o


# ---- read kernels ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("gs", list(GAMES))
def test_read_kernels_at_every_batch_size(gs):
    pool, L = pool_of(gs), _lib.lib()
    P, W, F, I = pool.P, pool.W, pool.F, pool.I
    for n in sizes(GAMES[gs]):
        perm = perm_for(n, n)
        b = pool.fill(perm)
        node = 4 * perm[:n]
        tails = tail_blobs(b, n)
        st = b._stream()
        what = "%s n=%d" % (gs, n)
        cur, term, rets = Guarded(n, 1, torch.int8, -99), Guarded(n, 1, torch.uint8, SENT8), out32(n, P)
        _lib.check(L.b2s_status(b._h, cur.ptr, term.ptr, rets.ptr, n, st))
        assert cur.intact() and term.intact() and rets.intact(), what
        np.testing.assert_array_equal(cur.rows()[:, 0], pool.cur[node], err_msg=what)
        np.testing.assert_array_equal(term.rows()[:, 0], pool.term[node], err_msg=what)
        np.testing.assert_array_equal(rets.rows(), pool.rets[node], err_msg=what)      # bits: the sign of zero included

        mask = out32(n, W)
        _lib.check(L.b2s_legal_mask(b._h, mask.ptr, n, st))
        assert mask.intact(), what
        np.testing.assert_array_equal(mask.rows(), pool.words[node], err_msg=what)

        most = int(pool.count[node].max())
        for stride in sorted({pool.width, max(1, most // 2)}):
            acts, counts = Guarded(n, stride, torch.int16, SENT16), out32(n, 1)
            _lib.check(L.b2s_legal_list(b._h, acts.ptr, counts.ptr, stride, n, st))
            assert acts.intact() and counts.intact(), (what, stride)
            np.testing.assert_array_equal(counts.rows()[:, 0], pool.count[node], err_msg=what)
            # rows cut at the stride; slots past a lane's count untouched
            np.testing.assert_array_equal(acts.rows(), pool.legal[node, :stride], err_msg="%s stride %d" % (what, stride))

        for which, size, table, fn in ((0, F, pool.obs, L.b2s_observation), (1, I, pool.info, L.b2s_information_state)):
            if not size:
                continue
            for player in list(range(P)) + [-1]:
                # player -1: the player to move, player 0 at chance nodes and terminal states
                pl = np.where(pool.cur[node] >= 0, pool.cur[node], 0) if player < 0 else np.full(n, player)
                want = table[node, pl]
                for off in range(4):
                    out = out32(n, size, offset=off)
                    _lib.check(fn(b._h, player, out.ptr, n, st))
                    assert out.intact(), (what, which, player, off)
                    np.testing.assert_array_equal(out.rows().view(np.float32), want,
                                                  err_msg="%s tensor %d player %d offset %d" % (what, which, player, off))
        assert tail_blobs(b, n) == tails, what
        assert b.error_count()[0] == 0


# ---- write kernels -----------------------------------------------------------------------------------------------------------

def entries(pool):
    e = ["apply", "step", "step_mask_only", "step_no_mask", "step_host"]
    if pool.wld():
        e += ["compact4", "compact4_mask"]
        if pool.A < 255:
            e += ["compact1", "compact1_mask"]
    return e


def run_entry(pool, b, entry, acts, n, pin=False, bufs=None):
    """One stepping call on lanes [0, n) of b; returns the fused outputs as numpy (None where the entry has none) after
    checking their guards.  Host buffers are pinned when `pin`; `bufs` (a dict) keeps them for the next call."""
    L, st = _lib.lib(), b._stream()
    P, W = pool.P, pool.W
    out = {"words": None, "term": None, "rets": None, "status": None}
    bufs = {} if bufs is None else bufs

    def Host(key, width, dtype, sentinel):
        if key not in bufs:
            bufs[key] = Guarded(n, width, dtype, sentinel, device="cpu", pin=pin)
        return bufs[key]

    if entry == "apply":
        a = torch.from_numpy(acts).cuda()
        b.apply_actions(a, n=n)
    elif entry in ("step", "step_mask_only", "step_no_mask"):
        a = torch.from_numpy(acts).cuda()
        mask = out32(n, W) if entry in ("step", "step_mask_only") else None
        term = Guarded(n, 1, torch.uint8, SENT8) if entry in ("step", "step_no_mask") else None
        rets = out32(n, P) if entry in ("step", "step_no_mask") else None
        _lib.check(L.b2s_step_fused(b._h, a.data_ptr(), mask.ptr if mask else None, term.ptr if term else None,
                                    rets.ptr if rets else None, n, st))
        torch.cuda.synchronize()
        for k, g in (("words", mask), ("term", term), ("rets", rets)):
            if g is not None:
                assert g.intact(), (entry, k)
                out[k] = g.rows()[:, 0] if k == "term" else g.rows()
    elif entry == "step_host":
        a = Host("a4", 1, torch.int32, -1)
        a.view().copy_(torch.from_numpy(acts[:n]))
        mask = Host("mask", W, torch.int32, SENT32)
        term = Host("term", 1, torch.uint8, SENT8)
        rets = Host("rets", P, torch.int32, SENT32)
        _lib.check(L.b2s_step_fused_host(b._h, a.ptr, mask.ptr, term.ptr, rets.ptr, n))
        for k, g in (("words", mask), ("term", term), ("rets", rets)):
            assert g.intact(), (entry, k)
            out[k] = g.rows()[:, 0] if k == "term" else g.rows()
    else:                                                          # compact{1,4}[_mask]
        ab = int(entry[7])
        if ab == 1:
            a = Host("a1", 1, torch.uint8, 0xFF)
            a.view().copy_(torch.from_numpy(np.where(acts[:n] < 0, 255, acts[:n]).astype(np.uint8)))
        else:
            a = Host("a4", 1, torch.int32, -1)
            a.view().copy_(torch.from_numpy(acts[:n]))
        status = Host("status", 1, torch.uint8, SENT8)
        mask = Host("mask", W, torch.int32, SENT32) if entry.endswith("mask") else None
        _lib.check(L.b2s_step_fused_host_compact(b._h, a.ptr, ab, status.ptr, mask.ptr if mask else None, n))
        assert status.intact(), entry
        out["status"] = status.rows()[:, 0]
        if mask is not None:
            assert mask.intact(), entry
            out["words"] = mask.rows()
    return out


def check_step(pool, b, entry, out, n, node, rejected, what):
    """Fused outputs and the lanes' next state against the tables; the error record against the rejected lanes."""
    cnt, first = b.error_count()
    assert cnt == len(rejected), (what, cnt, len(rejected))
    assert first == (int(rejected[0]) if len(rejected) else -1), (what, first)
    o = assert_state(pool, b, n, node, what)
    for k, table in (("words", pool.words), ("term", pool.term), ("rets", pool.rets), ("status", pool.status)):
        if out[k] is not None:
            np.testing.assert_array_equal(out[k], table[node], err_msg="%s fused %s" % (what, k))
    # a rejected lane's fused outputs are what status() / legal_actions_mask_words() then report
    for k in ("words", "term", "rets"):
        if out[k] is not None and len(rejected):
            np.testing.assert_array_equal(out[k][rejected], o[k][rejected], err_msg="%s rejected %s" % (what, k))


@pytest.mark.parametrize("gs", list(GAMES))
def test_write_kernels_at_every_batch_size(gs):
    pool = pool_of(gs)
    for n in sizes(GAMES[gs]):
        perm = perm_for(n, n + 1)
        b = pool.fill(perm)
        tails = tail_blobs(b, n)
        for e, entry in enumerate(entries(pool)):
            acts, node, rejected = pool.actions(perm, n, seed=n * 31 + e)
            pool.fill(perm, b)
            what = "%s n=%d %s" % (gs, n, entry)
            out = run_entry(pool, b, entry, acts, n)
            check_step(pool, b, entry, out, n, node, rejected, what)
            assert tail_blobs(b, n) == tails, what


# ---- host-buffer paths -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("gs", ["breakthrough", "go(board_size=9)"])
def test_host_step_graph_path(gs):
    """Pinned buffers and n >= 65536: the upload -> kernel -> download pipeline is captured once and replayed."""
    pool, L = pool_of(gs), _lib.lib()
    n = (1 << 16) + 37
    perm = perm_for(n, 5)
    b = pool.fill(perm)
    tails = tail_blobs(b, n)
    deltas = []
    for entry in ("step_host", "compact4_mask"):
        bufs = {}
        for rep in range(2):          # the first call captures the graph, the second replays it (same buffers, same n)
            acts, node, rejected = pool.actions(perm, n, seed=rep)
            pool.fill(perm, b)
            g0 = L.b2s_host_graph_launches()
            out = run_entry(pool, b, entry, acts, n, pin=True, bufs=bufs)
            deltas.append(L.b2s_host_graph_launches() - g0)
            check_step(pool, b, entry, out, n, node, rejected, "%s graph %s %d" % (gs, entry, rep))
            assert tail_blobs(b, n) == tails
    assert deltas == [1, 1, 1, 1], deltas


@pytest.mark.parametrize("gs", ["connect_four", "hex(board_size=5)", "go(board_size=9)", "othello"])
def test_host_step_zero_copy_path(gs):
    """Pinned, 16-byte aligned uint8 buffers, n >= 4096, no mask words: the kernel reads and writes host memory itself."""
    pool, L = pool_of(gs), _lib.lib()
    n = 4096 + 33 + 256 * GAMES[gs]           # a ragged last block
    perm = perm_for(n, 6)
    b = pool.fill(perm)
    tails = tail_blobs(b, n)
    acts, node, rejected = pool.actions(perm, n, seed=2)
    a = Guarded(n, 1, torch.uint8, 0xFF, device="cpu", pin=True)
    a.view().copy_(torch.from_numpy(np.where(acts[:n] < 0, 255, acts[:n]).astype(np.uint8)))
    status = Guarded(n, 1, torch.uint8, SENT8, device="cpu", pin=True)
    assert a.ptr % 16 == 0 and status.ptr % 16 == 0
    z0, g0 = L.b2s_host_zero_copy_steps(), L.b2s_host_graph_launches()
    _lib.check(L.b2s_step_fused_host_compact(b._h, a.ptr, 1, status.ptr, None, n))
    assert L.b2s_host_zero_copy_steps() - z0 == 1 and L.b2s_host_graph_launches() == g0
    assert status.intact()
    check_step(pool, b, "zero-copy", {"words": None, "term": None, "rets": None, "status": status.rows()[:, 0]}, n, node,
               rejected, "%s zero-copy" % gs)
    assert tail_blobs(b, n) == tails


CHUNKED = r"""
import sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import test_gpu_batch_geometry as T
T.chunked_child(sys.argv[3], int(sys.argv[4]))
print("ok")
"""


def chunked_child(gs, n):
    """Body of test_chunked_host_step (in a process with B2S_HOST_CHUNKS=3): pageable buffers, so the stream path steps the
    batch in three sub-range views; compared with the tables and with the same step on the device entry point."""
    pool, L = pool_of(gs), _lib.lib()
    chunk = ((n + 2) // 3 + 1023) // 1024 * 1024
    bad_lane = 2 * chunk + 517                                    # in the third chunk
    perm = perm_for(n - TAIL, 9)
    perm[bad_lane] = int(np.nonzero((pool.bad >= 0) & ~pool.terminal_pool)[0][0])
    entries_ = ["step_host"] + (["compact4_mask"] if pool.wld() else [])
    host = pool.fill(perm)
    dev = pool.game.new_batch(n)
    for entry in entries_:
        acts, node, _ = pool.actions(perm, n, seed=4, illegal=False, terminal=False)
        acts[bad_lane] = pool.bad[perm[bad_lane]]
        node[bad_lane] = 4 * perm[bad_lane]
        pool.fill(perm, host)
        pool.fill(perm, dev)
        c0 = L.b2s_launch_count()
        out = run_entry(pool, host, entry, acts, n)
        assert L.b2s_launch_count() - c0 == 3, (entry, L.b2s_launch_count() - c0)     # one kernel per chunk
        check_step(pool, host, entry, out, n, node, np.array([bad_lane]), "%s chunked %s" % (gs, entry))
        m, t, r = dev.step(torch.from_numpy(acts).cuda())
        assert np.array_equal(m.cpu().numpy(), pool.words[node]) and np.array_equal(t.cpu().numpy(), pool.term[node])
        lanes = sorted({0, 1, chunk - 1, chunk, chunk + 1, 2 * chunk - 1, 2 * chunk, bad_lane, n - 1} |
                       set(np.random.RandomState(1).randint(0, n, size=24).tolist()))
        for lane in lanes:
            assert lane_key(host, lane) == lane_key(dev, lane), (entry, lane)
    # then random play: host and device entry points stay identical
    host._reset_errors()
    dev._reset_errors()
    width = pool.width
    g = torch.Generator(device="cuda").manual_seed(1)
    for step in range(6):
        words = dev.legal_actions_mask_words()
        bits = ((words.unsqueeze(-1) >> torch.arange(32, device="cuda", dtype=torch.int32)) & 1).reshape(n, -1)[:, :width]
        score = torch.rand(bits.shape, generator=g, device="cuda") * bits
        acts = torch.where(bits.any(1), score.argmax(1).to(torch.int32), torch.full((n,), -1, dtype=torch.int32, device="cuda"))
        out = run_entry(pool, host, "step_host", acts.cpu().numpy(), n)
        m, t, r = dev.step(acts)
        assert np.array_equal(out["words"], m.cpu().numpy()) and np.array_equal(out["term"], t.cpu().numpy())
        assert np.array_equal(out["rets"], r.cpu().numpy().view(np.int32)), step
    assert host.error_count() == dev.error_count() == (0, -1)
    for lane in lanes:
        assert lane_key(host, lane) == lane_key(dev, lane), lane


@pytest.mark.parametrize("gs", ["breakthrough", "leduc_poker(players=4)", "go(board_size=9)"])
def test_chunked_host_step(gs, tmp_path):
    # B2S_HOST_CHUNKS is read once per process
    script = tmp_path / "chunked.py"
    script.write_text(CHUNKED)
    env = dict(os.environ, B2S_HOST_CHUNKS="3")
    r = subprocess.run([sys.executable, str(script), ROOT, HERE, gs, str((1 << 18) + 4133)], capture_output=True, text=True,
                       env=env, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-4000:] + r.stderr[-4000:]


# ---- clones ------------------------------------------------------------------------------------------------------------------

def mid_game(gs, n, seed):
    """n lanes of device-only random play, lane i stopped after 40 + (i * 7) % 160 plies or at the end."""
    game = b2.load_game(gs)
    b = game.new_batch(n)
    rng = np.random.RandomState(seed)
    stop = 40 + (np.arange(n) * 7) % 160
    for ply in range(int(stop.max())):
        acts, counts = b.legal_actions_list()
        acts, counts = acts.cpu().numpy(), counts.cpu().numpy()
        a = np.full(n, -1, dtype=np.int32)
        live = (counts > 0) & (ply < stop)
        pick = (rng.random_sample(n) * np.maximum(counts, 1)).astype(np.int64)
        a[live] = acts[np.arange(n), pick][live]
        b.apply_actions(torch.from_numpy(a).cuda())
    assert b.error_count()[0] == 0
    return game, b


@pytest.mark.parametrize("gs", ["go(board_size=9)", "go", "breakthrough"])
def test_clones_carry_the_whole_lane(gs):
    n, cap = 100, 140
    game, src = mid_game(gs, n, seed=3)
    keys = [lane_key(src, i) for i in range(n)]
    blank_batch = game.new_batch(1)
    blank = lane_key(blank_batch, 0)
    longest = max(range(n), key=lambda i: len(keys[i]))     # go: the longest history
    rng = np.random.RandomState(8)
    gather_idx = rng.permutation(n)[:97]
    cases = []
    d = game.new_batch(cap)
    d.copy_from(src, src_begin=5, dst_begin=37, count=41)
    cases.append(("copy", d, {37 + j: 5 + j for j in range(41)}))
    d = game.new_batch(cap)
    d.broadcast_from(src, longest, dst_begin=31, count=66)
    cases.append(("broadcast", d, {lane: longest for lane in range(31, 97)}))
    d = game.new_batch(cap)
    idx = torch.from_numpy(gather_idx.astype(np.int64)).cuda()
    _lib.check(_lib.lib().b2s_gather_states(d._h, src._h, C.c_void_p(idx.data_ptr()), len(gather_idx), d._stream()))
    cases.append(("gather", d, {i: int(s) for i, s in enumerate(gather_idx)}))
    for name, d, where in cases:
        assert d.error_count()[0] == 0, name
        for lane in range(cap):
            want = keys[where[lane]] if lane in where else blank
            assert lane_key(d, lane) == want, (gs, name, lane)
        # cloned lanes play on as their sources: a batch set lane by lane from the source blobs rolls out identically
        ref = game.new_batch(cap)
        for lane, s in where.items():
            ref.set_state_blob(lane, src.state_blob(s))
        r1, p1 = d.rollout(0xBEEF, lane_offset=11)
        r2, p2 = ref.rollout(0xBEEF, lane_offset=11)
        assert torch.equal(p1, p2) and torch.equal(r1, r2), (gs, name)
        assert int(p1.max()) > 0
