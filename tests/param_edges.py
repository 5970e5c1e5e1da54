"""The accepted parameter range of every rule core (make_cfg in open_spiel_b200/csrc/rules_*.cuh), sampled where the packed
layouts change code path, and the first shape past each limit.  Shared by test_gpu_param_edges.py (the device kernels),
test_param_edges_host.py (the host build of the rule cores) and test_param_edges_reference.py (the oracle against the
unmodified reference, through golden/param_edges_reference.json).  Test infrastructure.

ACCEPTED is a list of (game string, lanes): lanes is the device lock-step's lane count, ragged and past one warp except on the
largest boards.  REJECTED must fail load_game and b2s_batch_create.  SEARCH lists one or two edge shapes per deterministic
game for the device MCTS and AlphaBetaSearch; SEARCH_REJECTED / MCTS_REJECTED are accepted games too long for the searches'
path stacks, which those searches must refuse."""
import ctypes as C

import oracle_lib
from oracle_lib import OracleGame, OracleState

# connect_four: rows, columns, x_in_row >= 1; (rows+1)*columns <= 64 (one column-major word with a sentinel row) and
# columns <= 32 (the legal mask is one 32-bit word).  Path switches: the outcome cache in bits 62-63 of the key needs
# (rows+1)*columns <= 62; the multiply-gathers of the legal mask and of the observation rows need columns <= 24; unpack's
# fill[4] / fill[5] run on columns taller than 15 / 31 stones; has_line's four-in-a-row fast path shifts by up to
# 2*(rows+2), the general loop stops at i*d >= 64.
_C4_SHAPES = [
    (30, 2), (1, 31),                                           # (rows+1)*cols = 62: the last shapes with the outcome cache
    (2, 21), (6, 9), (8, 7), (20, 3), (62, 1),                  # 63
    (1, 32), (3, 16), (7, 8), (15, 4), (31, 2), (63, 1),        # 64: no spare bit at all
    (1, 24), (1, 25),                                           # the last gathered row and the first loop fallback
    (16, 3), (40, 1),                                           # tall columns: fill[4], and fill[5] past 32 stones
    (29, 2),                                                    # the tallest board on has_line's fast path
]
CONNECT_FOUR = ["connect_four(rows=%d,columns=%d)" % rc for rc in _C4_SHAPES] + [
    "connect_four(x_in_row=1)", "connect_four(x_in_row=2)", "connect_four(x_in_row=3)", "connect_four(x_in_row=5)",
    "connect_four(x_in_row=8)",                                 # longer than both sides: every game is a draw
    "connect_four(rows=20,columns=3,x_in_row=5)",               # the general loop at i*d = 4*21 >= 64 (diagonals cut)
    "connect_four(rows=31,columns=2,x_in_row=3)",               # 2*33 >= 64 on the diagonal
    "connect_four(rows=62,columns=1,x_in_row=3)",
    "connect_four(rows=8,columns=7,egocentric_obs_tensor=True)",
]

# breakthrough: rows, columns >= 2, rows*columns <= 64.
BREAKTHROUGH = ["breakthrough(rows=%d,columns=%d)" % rc for rc in
                [(2, 2), (2, 32), (32, 2), (4, 16), (16, 4), (5, 12), (6, 10), (7, 9), (21, 3)]]

# hex: num_rows, num_cols >= 2 (on one row or column the reference never ends a game: its edge tests, hex.cc:122-126 and
# 146-150, give a stone on both edges only one), num_cols*num_rows <= 121, num_cols <= 63 (b_shl / b_shr by cols - 1 and
# cols + 1 on the 128-bit board); swap needs num_cols <= num_rows (hex.cc:238), plain_obs_tensor num_cols >= num_rows.
HEX = ["hex(num_rows=%d,num_cols=%d)" % rc for rc in
       [(2, 2), (2, 60), (60, 2), (3, 40), (8, 8), (5, 13), (13, 5), (10, 12), (12, 10)]] + [
    "hex(num_rows=11,num_cols=11,swap=True)",                   # the swap action is bit 121: mask word 3
    "hex(num_rows=60,num_cols=2,swap=True)",
    "hex(num_rows=2,num_cols=60,plain_obs_tensor=True)",
]

# go: board_size 2..19 (2..9 on the 128-bit core, 10..19 on the 384-bit one), max_game_length <= 1000, handicap >= 2 only
# on boards of 16 and more (the stones sit on 19x19 coordinates up to row 16).
GO = ["go(board_size=%d)" % n for n in range(2, 20)] + [
    "go(board_size=%d,handicap=%d)" % (n, h) for n in (16, 17, 18) for h in (2, 5, 9)] + [
    "go(board_size=7,handicap=1)", "go(board_size=19,handicap=0)", "go(board_size=13,handicap=1)",
    "go(board_size=9,max_game_length=1)", "go(board_size=19,max_game_length=2)", "go(board_size=4,max_game_length=1000)",
    "go(board_size=9,max_game_length=174)",                     # the longest game the go <= 9 searches hold
]

# mnk: m (columns), n (rows) 1..15 on a 256-bit board; k >= 1.
MNK = ["mnk(m=%d,n=%d,k=%d)" % v for v in
       [(1, 15, 3), (15, 1, 3), (8, 8, 4), (5, 13, 4), (11, 12, 5), (13, 15, 5), (15, 15, 5),
        (6, 6, 1), (6, 6, 2), (7, 5, 7), (7, 5, 8), (15, 15, 15), (15, 15, 16)]]

Y = ["y(board_size=%d)" % n for n in range(1, 12)]                                                  # 1..11
HAVANNAH = ["havannah(board_size=%d%s)" % (n, s) for n in range(1, 9) for s in ("", ",swap=True")]  # 1..8
KUHN = ["kuhn_poker(players=%d)" % p for p in range(2, 6)]                                          # 2..5
LEDUC = ["leduc_poker(players=%d,starting_player=%d)" % (p, s) for p in range(2, 5) for s in range(p)]   # 2..4
OTHER = ["othello", "tic_tac_toe"]

INFO_STATE = set(KUHN + LEDUC)


def _lanes(gs):
    """Device lock-step lanes: ragged and past one warp; fewer on the largest boards."""
    if gs.startswith("go"):
        n = int(gs.split("board_size=")[1].split(",")[0].rstrip(")"))
        return 97 if n <= 5 else 45 if n <= 9 else 19 if "max_game_length=" in gs else 13
    if gs.startswith(("mnk(m=15,n=15", "mnk(m=13", "hex(num_rows=11", "havannah(board_size=8", "havannah(board_size=7")):
        return 45
    return 77 if gs.startswith(("kuhn", "leduc")) else 69


def host_lanes(gs, lanes):
    """Lanes of the host build's lock-step check."""
    return max(4, lanes // 6)


def reference_lanes(gs, lanes):
    """Lanes of the recorded reference digests (golden/param_edges_reference.json)."""
    return max(3, lanes // 8)


ACCEPTED = [(gs, _lanes(gs)) for gs in CONNECT_FOUR + BREAKTHROUGH + HEX + GO + MNK + Y + HAVANNAH + KUHN + LEDUC + OTHER]

REJECTED = [
    "connect_four(rows=12,columns=5)", "connect_four(rows=1,columns=33)", "connect_four(rows=64,columns=1)",
    "connect_four(rows=0)", "connect_four(columns=0)", "connect_four(x_in_row=0)",
    "breakthrough(rows=5,columns=13)", "breakthrough(rows=13,columns=5)", "breakthrough(rows=1,columns=8)",
    "breakthrough(rows=8,columns=1)",
    "hex(num_rows=2,num_cols=61)", "hex(num_rows=1,num_cols=64)", "hex(num_rows=11,num_cols=12)", "hex(num_rows=3,num_cols=1)",
    "hex(num_rows=1,num_cols=2)", "hex(num_rows=1,num_cols=63)", "hex(num_rows=1,num_cols=63,plain_obs_tensor=True)",
    "hex(num_rows=2,num_cols=3,swap=True)", "hex(num_rows=3,num_cols=2,plain_obs_tensor=True)",
    "go(board_size=20)", "go(board_size=1)", "go(board_size=15,handicap=2)", "go(board_size=9,max_game_length=1001)",
    "mnk(m=16,n=15)", "mnk(m=15,n=16)", "mnk(k=0)",
    "y(board_size=12)", "y(board_size=0)",
    "havannah(board_size=9)", "havannah(board_size=0)",
    "kuhn_poker(players=6)", "kuhn_poker(players=1)",
    "leduc_poker(players=5)", "leduc_poker(players=1)", "leduc_poker(starting_player=2)",
    "leduc_poker(players=3,starting_player=3)",
]

# (game string, trees, prefix plies, simulations) for one small device MCTS per deterministic game, on its layout edges and
# at the longest game its path stack holds (max_game_length + 2 == kMaxPath: go <= 9 at 174).
SEARCH = [
    ("connect_four(rows=31,columns=2)", 40, 20, 150), ("connect_four(rows=1,columns=32)", 40, 6, 150),
    ("connect_four(rows=40,columns=1)", 33, 10, 60),
    ("breakthrough(rows=2,columns=32)", 40, 0, 100), ("breakthrough(rows=7,columns=9)", 33, 8, 100),
    ("hex(num_rows=11,num_cols=11,swap=True)", 33, 1, 100), ("hex(num_rows=2,num_cols=60)", 33, 8, 100),
    ("go(board_size=9,max_game_length=174)", 33, 20, 40), ("go(board_size=2)", 40, 4, 100),
    ("mnk(m=15,n=15,k=16)", 33, 10, 60), ("mnk(m=1,n=15,k=3)", 40, 4, 150),
    ("y(board_size=11)", 33, 6, 80), ("y(board_size=1)", 8, 0, 20),
    ("havannah(board_size=8,swap=True)", 33, 1, 60), ("havannah(board_size=1)", 8, 0, 20),
    ("othello", 33, 20, 80), ("tic_tac_toe", 40, 2, 200),
]


class BoardTextOracle(OracleGame):
    """OracleGame whose states' text decodes on every board: breakthrough labels columns past the 26th with the bytes after
    'z', which are not UTF-8, and parity.lockstep formats the board into the message of every tensor comparison."""

    def new_initial_state(self):
        return _BoardTextState(self, oracle_lib.lib().orc_new_initial_state(self._g))


class _BoardTextState(OracleState):
    def _str(self, fn, *args):
        buf = C.create_string_buffer(4096)
        fn(self._s, *args, buf, 4096)
        return buf.value.decode(errors="backslashreplace")


def raw_params(gs):
    """(game id, b2s_params) of a game string without the validation of load_game: what a caller of the C ABI could pass."""
    from open_spiel_b200 import spiel
    from open_spiel_b200._lib import Params, lib
    name, p = spiel._parse_game_string(gs)
    cp = Params()
    lib().b2s_params_default(C.byref(cp))
    fields = spiel._PARAM_FIELDS[name]
    for k, v in p.items():
        if fields[k] == "komi":
            cp.komi = float(v)
        else:
            setattr(cp, fields[k], int(v))
    return lib().b2s_game_id(name.encode()), cp


# the first max_game_length past each search's path stack, and accepted shapes whose games are longer than it holds
# (breakthrough: kMaxPath 224, max_game_length 233 / 235 / 245)
SEARCH_REJECTED = ["go(board_size=9,max_game_length=175)", "go(board_size=2,max_game_length=175)",
                   "breakthrough(rows=16,columns=4)", "breakthrough(rows=21,columns=3)", "breakthrough(rows=32,columns=2)"]
MCTS_REJECTED = SEARCH_REJECTED + ["go(board_size=10,max_game_length=723)"]   # the 384-bit core's MCTS stack holds 722
