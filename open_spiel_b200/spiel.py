"""Host-side mirror of open_spiel::Game / State (open_spiel/spiel.h:301-1255) over the C ABI."""
import ctypes as C
import math
import re

import numpy as np
import torch

from . import _lib
from ._lib import B2SError, GameInfo, Params, check, lib

kChancePlayerId = -1      # spiel_globals.h:26-56
kTerminalPlayerId = -4
kInvalidAction = -1

_NAMES = ["tic_tac_toe", "connect_four", "breakthrough", "hex", "go", "kuhn_poker", "leduc_poker", "mnk", "othello", "y", "havannah"]


def registered_names():
    """Short names this library serves (cf. pyspiel.registered_names, pyspiel.cc:737)."""
    return list(_NAMES)


def _parse_game_string(s):
    """'go(board_size=9,komi=7.5)' -> ('go', {...}); grammar of game_parameters.cc GameParametersFromString."""
    s = s.strip()
    m = re.match(r"^([\w]+)(?:\((.*)\))?$", s)
    if not m:
        raise B2SError("cannot parse game string: " + s)
    name, body = m.group(1), m.group(2)
    params = {}
    if body:
        for kv in body.split(","):
            if not kv.strip():
                continue
            k, v = kv.split("=", 1)
            v = v.strip()
            if v in ("True", "true"):
                params[k.strip()] = True
            elif v in ("False", "false"):
                params[k.strip()] = False
            else:
                try:
                    params[k.strip()] = int(v)
                except ValueError:
                    try:
                        params[k.strip()] = float(v)
                    except ValueError:
                        params[k.strip()] = v
    return name, params


_PARAM_FIELDS = {
    "connect_four": {"rows": "rows", "columns": "columns", "x_in_row": "x_in_row",
                     "egocentric_obs_tensor": "egocentric_obs_tensor"},
    "breakthrough": {"rows": "rows", "columns": "columns"},
    "hex": {"board_size": "board_size", "num_cols": "columns", "num_rows": "rows", "swap": "swap",
            "plain_obs_tensor": "plain_obs_tensor"},
    "go": {"board_size": "board_size", "komi": "komi", "handicap": "handicap",
           "max_game_length": "max_game_length"},
    "kuhn_poker": {"players": "players"},
    "leduc_poker": {"players": "players", "starting_player": "starting_player"},
    "tic_tac_toe": {},
    "mnk": {"m": "columns", "n": "rows", "k": "x_in_row"},
    "othello": {},
    "y": {"board_size": "board_size"},
    "havannah": {"board_size": "board_size", "swap": "swap"},
}


def load_game(game_string, params=None):
    """pyspiel.load_game (pyspiel.cc:720-735 -> spiel.cc:255-297)."""
    name, p = _parse_game_string(game_string)
    if params:
        p.update(params)
    return Game(name, p)


class Game:
    """Mirror of open_spiel::Game for the seven device games."""

    def __init__(self, name, params=None, device=0):
        L = lib()
        self._name = name
        self._params = dict(params or {})
        gid = L.b2s_game_id(name.encode())
        if gid < 0:
            raise B2SError("Unknown game '%s'. Available games are: %s" % (name, ", ".join(_NAMES)))
        self._gid = gid
        self._cparams = Params()
        L.b2s_params_default(C.byref(self._cparams))
        fields = _PARAM_FIELDS[name]
        for k, v in self._params.items():
            if k not in fields:
                raise B2SError("Unknown parameter '%s' for game %s" % (k, name))   # spiel.cc:65-89
            if fields[k] == "komi":
                self._cparams.komi = float(v)
            else:
                setattr(self._cparams, fields[k], int(v))
        self._info = GameInfo()
        check(L.b2s_game_info_get(gid, C.byref(self._cparams), C.byref(self._info)))
        self.device = device

    # -- Game API (spiel.h:927-1190) --
    def get_type_short_name(self):
        return self._name

    def num_distinct_actions(self):
        return self._info.num_distinct_actions

    def num_players(self):
        return self._info.num_players

    def max_game_length(self):
        return self._info.max_game_length

    def max_chance_outcomes(self):
        return self._info.max_chance_outcomes

    def min_utility(self):
        return self._info.min_utility

    def max_utility(self):
        return self._info.max_utility

    def observation_tensor_size(self):
        return self._info.observation_tensor_size

    def observation_tensor_shape(self):
        return [d for d in self._info.obs_shape if d > 0]

    def information_state_tensor_size(self):
        return self._info.information_state_tensor_size

    def get_parameters(self):
        return dict(self._params)

    def new_initial_state(self):
        return State(self)

    def deserialize_state(self, text):
        """Game::DeserializeState (spiel.cc:757-791): replay a State::Serialize action list from the initial state."""
        from .serialization import deserialize_state
        return deserialize_state(self, text)

    def new_batch(self, n, device=None):
        return BatchedState(self, n, self.device if device is None else device)

    def __str__(self):
        if not self._params:
            return self._name + "()"
        return self._name + "(" + ",".join("%s=%s" % (k, self._params[k]) for k in sorted(self._params)) + ")"


class BatchedState:
    """`n` States of one game, struct-of-arrays in HBM.  The batched extension the kernels exist for.

    Tensor arguments/results are torch CUDA tensors on the batch's device; work is enqueued on the
    current torch stream.
    """

    def __init__(self, game, n, device=0):
        if not torch.cuda.is_available():
            raise B2SError("no CUDA device: open_spiel_b200 has no CPU fallback")
        self.game, self.n, self.device = game, int(n), int(device)
        self._h = C.c_void_p()
        check(lib().b2s_batch_create(game._gid, C.byref(game._cparams), self.n, self.device, C.byref(self._h)))
        self.info = game._info
        self._dev = torch.device("cuda", self.device)

    def __del__(self):
        try:
            if self._h:
                lib().b2s_batch_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self._dev).cuda_stream)

    def _n(self, n):
        return self.n if n is None else int(n)

    def reset(self, n=None):
        check(lib().b2s_reset(self._h, self._n(n), self._stream()))

    def apply_actions(self, actions, n=None):
        assert actions.dtype == torch.int32 and actions.is_cuda and actions.is_contiguous()
        check(lib().b2s_apply_actions(self._h, actions.data_ptr(), self._n(n), self._stream()))

    def legal_actions_mask_words(self, out=None, n=None):
        n = self._n(n)
        if out is None:
            out = torch.empty((n, self.info.mask_words), dtype=torch.int32, device=self._dev)
        check(lib().b2s_legal_mask(self._h, out.data_ptr(), n, self._stream()))
        return out

    def legal_actions_mask(self, n=None):
        """Dense 0/1 mask [n, A] as State::LegalActionsMask (spiel.cc:518-524) would give."""
        words = self.legal_actions_mask_words(n=n)
        width = max(self.info.num_distinct_actions, self.info.max_chance_outcomes)
        bits = torch.arange(32, device=self._dev, dtype=torch.int32)
        dense = ((words.unsqueeze(-1) >> bits) & 1).reshape(words.shape[0], -1)[:, :width]
        return dense

    def legal_actions_list(self, stride=None, n=None):
        n = self._n(n)
        stride = stride or max(self.info.num_distinct_actions, self.info.max_chance_outcomes)
        acts = torch.full((n, stride), -1, dtype=torch.int16, device=self._dev)
        counts = torch.empty((n,), dtype=torch.int32, device=self._dev)
        check(lib().b2s_legal_list(self._h, acts.data_ptr(), counts.data_ptr(), stride, n, self._stream()))
        return acts, counts

    def status(self, n=None):
        n = self._n(n)
        cur = torch.empty((n,), dtype=torch.int8, device=self._dev)
        term = torch.empty((n,), dtype=torch.uint8, device=self._dev)
        rets = torch.empty((n, self.info.num_players), dtype=torch.float32, device=self._dev)
        check(lib().b2s_status(self._h, cur.data_ptr(), term.data_ptr(), rets.data_ptr(), n, self._stream()))
        return cur, term, rets

    def observation_tensor(self, player=-1, out=None, n=None):
        n = self._n(n)
        if out is None:
            out = torch.empty((n, self.info.observation_tensor_size), dtype=torch.float32, device=self._dev)
        check(lib().b2s_observation(self._h, int(player), out.data_ptr(), n, self._stream()))
        return out

    def information_state_tensor(self, player=-1, out=None, n=None):
        n = self._n(n)
        if out is None:
            out = torch.empty((n, self.info.information_state_tensor_size), dtype=torch.float32, device=self._dev)
        check(lib().b2s_information_state(self._h, int(player), out.data_ptr(), n, self._stream()))
        return out

    def step(self, actions, mask_out=None, terminal_out=None, returns_out=None, n=None):
        """Fused ApplyAction + IsTerminal + Returns + next legal mask."""
        n = self._n(n)
        assert actions.dtype == torch.int32 and actions.is_cuda
        if mask_out is None:
            mask_out = torch.empty((n, self.info.mask_words), dtype=torch.int32, device=self._dev)
        if terminal_out is None:
            terminal_out = torch.empty((n,), dtype=torch.uint8, device=self._dev)
        if returns_out is None:
            returns_out = torch.empty((n, self.info.num_players), dtype=torch.float32, device=self._dev)
        check(lib().b2s_step_fused(self._h, actions.data_ptr(), mask_out.data_ptr(), terminal_out.data_ptr(),
                                   returns_out.data_ptr(), n, self._stream()))
        return mask_out, terminal_out, returns_out

    def step_host(self, actions_h, mask_h, terminal_h, returns_h, n=None):
        """Same step with HOST tensors (ideally pinned): H2D + kernel + D2H + sync inside the call."""
        n = self._n(n)
        check(lib().b2s_step_fused_host(self._h, actions_h.data_ptr(),
                                        mask_h.data_ptr() if mask_h is not None else None,
                                        terminal_h.data_ptr() if terminal_h is not None else None,
                                        returns_h.data_ptr() if returns_h is not None else None, n))

    def step_host_compact(self, actions_h, status_h, mask_h=None, n=None):
        """b2s_step_fused_host_compact: uint8 (0xFF = skip) or int32 actions in, one status byte per lane out
        (bit 7 terminal; terminal: bits 0-1 outcome 0 draw / 1 player 0 / 2 player 1; else bits 0-6 the legal mask when
        the game has <= 7 actions); mask_h optionally receives the full mask words."""
        n = self._n(n)
        ab = {torch.uint8: 1, torch.int32: 4}[actions_h.dtype]
        check(lib().b2s_step_fused_host_compact(self._h, actions_h.data_ptr(), ab, status_h.data_ptr(),
                                                mask_h.data_ptr() if mask_h is not None else None, n))

    def rollout(self, seed, lane_offset=0, n=None):
        n = self._n(n)
        rets = torch.empty((n, self.info.num_players), dtype=torch.float32, device=self._dev)
        plies = torch.empty((n,), dtype=torch.int32, device=self._dev)
        check(lib().b2s_rollout(self._h, int(seed), int(lane_offset), n, rets.data_ptr(), plies.data_ptr(), self._stream()))
        return rets, plies

    def record_trajectories(self, seed, lane_offset=0, n=None, max_unroll_length=None, include_full_observations=True):
        """Batched algorithms::RecordBatchedTrajectory (trajectories.cc:98-200) with uniform-random policies: plays
        every lane from its current state to the end and returns a BatchedTrajectory of device tensors."""
        from ._lib import TrajectoryOut
        n = self._n(n)
        T = int(max_unroll_length) if max_unroll_length else self.info.max_game_length
        info, dev = self.info, self._dev
        F = info.information_state_tensor_size if info.information_state_tensor_size > 0 else info.observation_tensor_size
        tm = {      # time-major device buffers
            "observations": torch.empty((T, n, F), dtype=torch.float32, device=dev) if include_full_observations else None,
            "legal_mask": torch.empty((T, n, info.mask_words), dtype=torch.int32, device=dev),
            "actions": torch.empty((T, n), dtype=torch.int32, device=dev),
            "player_ids": torch.empty((T, n), dtype=torch.int8, device=dev),
            "valid": torch.empty((T, n), dtype=torch.uint8, device=dev),
            "next_is_terminal": torch.empty((T, n), dtype=torch.uint8, device=dev),
            "rewards": torch.empty((n, info.num_players), dtype=torch.float32, device=dev),
            "lengths": torch.empty((n,), dtype=torch.int32, device=dev),
        }
        out = TrajectoryOut(**{k: (v.data_ptr() if v is not None else None) for k, v in tm.items()})
        check(lib().b2s_record_trajectories(self._h, int(seed), int(lane_offset), n, T, C.byref(out), self._stream()))
        return BatchedTrajectory(n, T, info.num_distinct_actions, tm)

    def error_count(self):
        cnt, first = C.c_int64(), C.c_int64()
        check(lib().b2s_error_count(self._h, C.byref(cnt), C.byref(first), self._stream()))
        return cnt.value, first.value

    def check_errors(self):
        cnt, first = self.error_count()
        if cnt:
            raise B2SError("%d lane(s) rejected an illegal action (first lane %d)" % (cnt, first))

    def state_blob(self, idx):
        size = self.info.state_bytes + self.info.history_bytes
        buf = (C.c_uint8 * size)()
        check(lib().b2s_state_get(self._h, int(idx), buf, size))
        return bytes(buf)

    def set_state_blob(self, idx, blob):
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        check(lib().b2s_state_set(self._h, int(idx), buf, len(blob)))

    def broadcast_from(self, src_batch, src_lane, dst_begin=0, count=None):
        count = self.n - dst_begin if count is None else count
        check(lib().b2s_broadcast_state(self._h, dst_begin, count, src_batch._h, int(src_lane), self._stream()))


    def copy_from(self, src_batch, src_begin=0, dst_begin=0, count=None):
        count = min(self.n - dst_begin, src_batch.n - src_begin) if count is None else count
        check(lib().b2s_copy_states(self._h, dst_begin, src_batch._h, src_begin, count, self._stream()))


class State:
    """Mirror of open_spiel::State (scalar API) backed by a one-lane device batch.

    Every call launches a kernel and synchronises: this adapter exists for API/parity tests and for code
    that is written against the scalar State interface; throughput comes from BatchedState.
    """

    def __init__(self, game, _batch=None, _history=None):
        self._game = game
        self._b = _batch if _batch is not None else BatchedState(game, 1, game.device)
        self._history = list(_history or [])      # [(player, action)] as State::history_ (spiel.h:911)
        self._act = torch.empty((1,), dtype=torch.int32, device=self._b._dev)

    def get_game(self):
        return self._game

    def current_player(self):
        cur, _, _ = self._b.status()
        return int(cur.item())

    def is_terminal(self):
        _, term, _ = self._b.status()
        return bool(term.item())

    def is_chance_node(self):
        return self.current_player() == kChancePlayerId

    def legal_actions(self, player=None):
        cur = self.current_player()
        if cur == kTerminalPlayerId or (player is not None and player != cur):
            return []
        acts, counts = self._b.legal_actions_list()
        k = int(counts.item())
        return [int(a) for a in acts[0, :k].tolist()]

    def legal_actions_mask(self, player=None):
        cur = self.current_player()
        width = self._game.num_distinct_actions() if cur != kChancePlayerId else self._game.max_chance_outcomes()
        if player is not None and player != cur:
            return [0] * width
        return [int(v) for v in self._b.legal_actions_mask()[0, :width].tolist()]

    def apply_action(self, action):
        if action == kInvalidAction:
            raise B2SError("ApplyAction: action == kInvalidAction")      # spiel.cc:443
        player = self.current_player()
        self._act[0] = int(action)
        self._b.apply_actions(self._act)
        cnt, _ = self._b.error_count()
        if cnt:
            self._b._reset_errors()
            raise B2SError("illegal action %d for state\n%s" % (action, self))
        self._history.append((player, int(action)))

    def returns(self):
        _, _, rets = self._b.status()
        return [float(v) for v in rets[0].tolist()]

    def rewards(self):
        # default State::Rewards (spiel.h:489-495): zeros until terminal, then Returns()
        if self.is_terminal():
            return self.returns()
        return [0.0] * self._game.num_players()

    def player_return(self, player):
        return self.returns()[player]

    def observation_tensor(self, player=None):
        if player is None:
            player = max(self.current_player(), 0)
        return self._b.observation_tensor(player)[0].cpu().numpy()

    def information_state_tensor(self, player=None):
        if player is None:
            player = max(self.current_player(), 0)
        return self._b.information_state_tensor(player)[0].cpu().numpy()

    def information_state_string(self, player=None):
        """State::InformationStateString (kuhn_poker.cc:109-166, leduc_poker.cc:198-239), rebuilt on the host from the
        device's information-state tensor (open_spiel_b200/serialization.py)."""
        from .serialization import INFORMATION_STATE_STRING
        f = INFORMATION_STATE_STRING.get(self._game._name)
        if f is None:
            raise B2SError("%s provides no information state string" % self._game._name)
        return f(self.information_state_tensor(player))

    def chance_outcomes(self):
        """State::ChanceOutcomes: kuhn / leduc deal uniformly over the remaining cards (kuhn_poker.cc:329-337,
        leduc_poker.cc:546-571)."""
        if not self.is_chance_node():
            raise B2SError("chance_outcomes() at a non-chance node")
        la = self.legal_actions()
        return [(a, 1.0 / len(la)) for a in la]

    def history(self):
        return [a for _, a in self._history]

    def full_history(self):
        return list(self._history)

    def move_number(self):
        return len(self._history)

    def clone(self):
        nb = BatchedState(self._game, 1, self._game.device)
        nb.broadcast_from(self._b, 0, 0, 1)
        return State(self._game, nb, self._history)

    def child(self, action):
        c = self.clone()
        c.apply_action(action)
        return c

    def serialize(self):
        """State::Serialize default format: one action per line (spiel.cc:411-430)."""
        return "".join("%d\n" % a for _, a in self._history)

    def __str__(self):
        return "<b200 %s state, history=%s>" % (self._game.get_type_short_name(), self.history())


def _reset_errors(self):
    # clear the error counter without touching states: reset zero lanes
    check(lib().b2s_reset(self._h, 0, self._stream()))


BatchedState._reset_errors = _reset_errors


class BatchedTrajectory:
    """Mirror of algorithms::BatchedTrajectory (trajectories.h:34-75).  The fields are [B, T, ...] views of the
    time-major device buffers the recorder fills (no copy): observations, legal_mask (bit-packed; legal_actions()
    expands it to the reference's [B, T, A] 0/1 ints), actions, player_ids, valid, next_is_terminal; rewards is
    [B, num_players] and lengths [B]."""

    def __init__(self, batch_size, T, num_actions, tm):
        self.batch_size, self.max_trajectory_length, self._A = batch_size, T, num_actions
        self.time_major = tm
        for k in ("observations", "legal_mask", "actions", "player_ids", "valid", "next_is_terminal"):
            setattr(self, k, tm[k].transpose(0, 1) if tm[k] is not None else None)
        self.rewards, self.lengths = tm["rewards"], tm["lengths"]

    def legal_actions(self):
        """[B, T, A] int32 0/1 as BatchedTrajectory::legal_actions (padding rows are all ones)."""
        shifts = torch.arange(32, device=self.legal_mask.device, dtype=torch.int32)
        bits = (self.legal_mask.unsqueeze(-1) >> shifts) & 1            # [B, T, W, 32]
        return bits.reshape(*self.legal_mask.shape[:2], -1)[..., :self._A].to(torch.int32)

    def player_policies(self):
        """[B, T, A] float64: the uniform policy that generated the actions (padding rows are all ones)."""
        la = self.legal_actions().to(torch.float64)
        return la / la.sum(-1, keepdim=True).clamp_(min=1) * self.valid.unsqueeze(-1) + la * (1 - self.valid.unsqueeze(-1))


class StepType:
    """rl_environment.StepType values as step_type holds them."""
    FIRST = 0
    MID = 1
    LAST = 2


class ObservationType:
    """rl_environment.ObservationType (rl_environment.py:78-81); VectorEnv also takes the reference's enum members."""
    INFORMATION_STATE = 0
    OBSERVATION = 1


class VectorTimeStep:
    """The time steps of all envs (rl_environment.TimeStep of each lane, stacked): info_state [n, P, F] float32,
    legal_actions_mask [n, A] bool (the player to move's; all False at LAST), current_player [n] int8, rewards [n, P]
    float32 (0 at FIRST where the reference has None), discounts [n, P] float32 (0 at LAST, `discount` otherwise, also at
    FIRST where the reference has None), step_type [n] uint8 (StepType).  Views of the env's buffers, which the next
    reset() / step() overwrites."""

    def __init__(self, info_state, legal_actions_mask, current_player, rewards, discounts, step_type):
        self.info_state, self.legal_actions_mask, self.current_player = info_state, legal_actions_mask, current_player
        self.rewards, self.discounts, self.step_type = rewards, discounts, step_type

    def first(self):
        return self.step_type == StepType.FIRST

    def last(self):
        return self.step_type == StepType.LAST


class VectorEnv:
    """rl_environment.Environment over `num_envs` lanes, stepped as vector_env.SyncVectorEnv (b2s_env_*): one reset() or
    step() is a fixed set of kernel launches on the current torch stream with no host synchronisation, so `policy
    forward + env.step` can be captured into a torch.cuda.CUDAGraph.  Chance nodes are sampled on the device from a
    Philox stream keyed by (seed, lane + lane_offset, call number) instead of the reference's numpy ChanceEventSampler.
    observation_type None = information state when the game has one, else observation (rl_environment.py:228-241).
    env.batch is the underlying BatchedState."""

    def __init__(self, game, num_envs, seed=0, observation_type=None, discount=1.0, lane_offset=0, device=0):
        from ._lib import EnvConfig, EnvOut
        if isinstance(game, str):
            game = load_game(game)
        self.game, self.num_envs, self.discount = game, int(num_envs), float(discount)
        self.batch = BatchedState(game, self.num_envs, device)
        info, dev, n = self.batch.info, self.batch._dev, self.num_envs
        kind = getattr(observation_type, "name", observation_type)
        which = {None: -1, ObservationType.OBSERVATION: 0, "OBSERVATION": 0,
                 ObservationType.INFORMATION_STATE: 1, "INFORMATION_STATE": 1}.get(kind)
        if which is None:
            raise B2SError("VectorEnv: unknown observation_type %r" % (observation_type,))
        self._h = C.c_void_p()
        check(lib().b2s_env_create(self.batch._h, C.byref(EnvConfig(int(seed), int(lane_offset), which, 0)), C.byref(self._h)))
        if which == -1:
            which = 1 if info.information_state_tensor_size > 0 else 0
        F = info.information_state_tensor_size if which == 1 else info.observation_tensor_size
        P, A = info.num_players, info.num_distinct_actions
        self._obs = torch.empty((P, n, F), dtype=torch.float32, device=dev)     # player-major, as the kernels write it
        self._mask_words = torch.empty((n, info.mask_words), dtype=torch.int32, device=dev)
        self._rewards = torch.empty((n, P), dtype=torch.float32, device=dev)
        self._done = torch.empty((n,), dtype=torch.uint8, device=dev)
        self._step_type = torch.empty((n,), dtype=torch.uint8, device=dev)
        self._cur = torch.empty((n,), dtype=torch.int8, device=dev)
        self._mask = torch.empty((n, A), dtype=torch.bool, device=dev)
        self._discounts = torch.empty((n, P), dtype=torch.float32, device=dev)
        self._bits = torch.arange(32, dtype=torch.int32, device=dev)
        self._out = EnvOut(self._obs.data_ptr(), self._mask_words.data_ptr(), self._rewards.data_ptr(), self._done.data_ptr(),
                           self._step_type.data_ptr(), self._cur.data_ptr())
        self._started = False
        self.time_step = VectorTimeStep(self._obs.permute(1, 0, 2), self._mask, self._cur, self._rewards, self._discounts,
                                        self._step_type)

    def __del__(self):
        try:
            if self._h:
                lib().b2s_env_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _finish(self):
        n, A = self.num_envs, self._mask.shape[1]
        bits = (self._mask_words.unsqueeze(-1) >> self._bits) & 1
        self._mask.copy_(bits.reshape(n, -1)[:, :A])
        torch.mul((self._step_type != StepType.LAST).unsqueeze(1).expand_as(self._discounts), self.discount, out=self._discounts)
        return self.time_step

    def reset(self):
        """SyncVectorEnv.reset(): Environment.reset of every env.  Returns the VectorTimeStep (all FIRST)."""
        check(lib().b2s_env_reset(self._h, self.num_envs, C.byref(self._out), self.batch._stream()))
        self._started = True
        return self._finish()

    def step(self, actions, reset_if_done=False):
        """SyncVectorEnv.step(actions, reset_if_done): returns (time_step, reward [n, P], done [n] bool), the first three
        results of the reference (unreset_time_steps is not kept).  actions [n] is an integer CUDA tensor, -1 leaves an
        env untouched; envs at LAST ignore their action and start a new episode.  An env never reset is reset, as
        Environment.step does before its first reset()."""
        if not self._started:
            return self.reset(), self._rewards, self._done.view(torch.bool)
        if actions.dtype != torch.int32 or not actions.is_contiguous():
            actions = actions.to(torch.int32).contiguous()
        if not actions.is_cuda or actions.numel() != self.num_envs:
            raise B2SError("VectorEnv.step: actions must be a CUDA tensor of %d integers" % self.num_envs)
        check(lib().b2s_env_step(self._h, actions.data_ptr(), int(bool(reset_if_done)), self.num_envs, C.byref(self._out),
                                 self.batch._stream()))
        return self._finish(), self._rewards, self._done.view(torch.bool)


class ChildSelectionPolicy:
    """algorithms::ChildSelectionPolicy (mcts.h:148)."""
    UCT = 0
    PUCT = 1


def mcts_search(batch, max_simulations, uct_c=2.0, n_rollouts=1, solve=True, seed=0, tree_index_offset=0,
                n_trees=None, max_nodes_total=0, child_selection_policy=ChildSelectionPolicy.UCT, max_nodes_per_tree=0,
                max_wall_clock_time=0.0):
    """Batched MCTSBot.mcts_search (python/pybind11/bots.cc:129-149 -> algorithms/mcts.cc:353-467) over the lanes of
    `batch`.  Returns dict of device tensors: visits [n, A] int32, total_reward [n, A] float64, outcome_p0 [n, A]
    float32 (NaN = unproven), best_action [n] int32, sims_run [n] int32, gc_runs [n] int32.  max_nodes_per_tree is
    MCTSBot's node budget max_nodes_ (garbage collection as mcts.cc:441-482), max_wall_clock_time its time budget."""
    from ._lib import MctsConfig
    n = batch.n if n_trees is None else int(n_trees)
    A = batch.info.num_distinct_actions
    dev = batch._dev
    out = {
        "visits": torch.empty((n, A), dtype=torch.int32, device=dev),
        "total_reward": torch.empty((n, A), dtype=torch.float64, device=dev),
        "outcome_p0": torch.empty((n, A), dtype=torch.float32, device=dev),
        "best_action": torch.empty((n,), dtype=torch.int32, device=dev),
        "sims_run": torch.empty((n,), dtype=torch.int32, device=dev),
        "gc_runs": torch.empty((n,), dtype=torch.int32, device=dev),
    }
    cfg = MctsConfig(int(max_simulations), int(n_rollouts), int(bool(solve)), int(child_selection_policy), float(uct_c), int(seed),
                     int(tree_index_offset), int(max_nodes_total), int(max_nodes_per_tree), float(max_wall_clock_time),
                     out["gc_runs"].data_ptr())
    check(lib().b2s_mcts_search(batch._h, n, C.byref(cfg), out["visits"].data_ptr(), out["total_reward"].data_ptr(),
                                out["outcome_p0"].data_ptr(), out["best_action"].data_ptr(), out["sims_run"].data_ptr(),
                                batch._stream()))
    return out


def alpha_beta_search(batch, depth_limit=-1, maximizing_player=-1, max_nodes=0, n=None):
    """algorithms::AlphaBetaSearch (algorithms/minimax.cc:221-258) with no value function, from each of the first n lanes of
    `batch` (b2s_alpha_beta_search).  Returns a dict of device tensors [n]: value float64 (PlayerReturn(maximizing_player) of
    the solved root), best_action int32 (-1 for a terminal root), nodes int64 (child states generated) and status uint8
    (0 solved, 1 max_nodes ran out, 2 a non-terminal state at depth 0, 3 maximizing_player -1 on a terminal root).
    maximizing_player -1 is the root's current player; depth_limit -1 and max_nodes 0 are unlimited.  Enqueued on the
    current stream."""
    from ._lib import AlphaBetaConfig
    n = batch.n if n is None else int(n)
    dev = batch._dev
    out = {
        "value": torch.empty((n,), dtype=torch.float64, device=dev),
        "best_action": torch.empty((n,), dtype=torch.int32, device=dev),
        "nodes": torch.empty((n,), dtype=torch.int64, device=dev),
        "status": torch.empty((n,), dtype=torch.uint8, device=dev),
    }
    cfg = AlphaBetaConfig(int(depth_limit), int(maximizing_player), int(max_nodes))
    check(lib().b2s_alpha_beta_search(batch._h, n, C.byref(cfg), out["value"].data_ptr(), out["best_action"].data_ptr(),
                                      out["nodes"].data_ptr(), out["status"].data_ptr(), batch._stream()))
    return out


class MCTSEvalSearch:
    """MCTSBot.MCTSearch (algorithms/mcts.cc:353-467) with a caller-supplied evaluator over n roots at once, driven in rounds
    (b2s_mcts_eval_*): every step() advances all live trees until each needs an evaluation or finishes; the states to evaluate
    are lanes of `.leaves` (a BatchedState of the roots' game), flagged by the returned `pending` mask.  The next step() takes
    the answers: values [n, num_players] and priors [n, num_distinct_actions] (float64 device tensors, priors by action id;
    rows of lanes that are not pending and entries of illegal actions are ignored).  step(None, None) starts the search.
    With a deterministic evaluator the trees equal the reference MCTSBot's with that Evaluator (child shuffles on the
    position-keyed stream of mcts_search).  root_noise [n, A] (float64, optional) is the root's Dirichlet noise, mixed in as
    (1 - dirichlet_epsilon) * prior + dirichlet_epsilon * noise (see dirichlet_noise()).  max_wall_clock_time is not
    supported: the caller owns the loop and its time budget."""

    def __init__(self, roots_batch, max_simulations, uct_c=2.0, solve=True, seed=0, tree_index_offset=0, n_trees=None,
                 child_selection_policy=ChildSelectionPolicy.UCT, max_nodes_per_tree=0, max_nodes_total=0, root_noise=None,
                 dirichlet_epsilon=0.0, leaves=None, max_wall_clock_time=0.0):
        from ._lib import MctsEvalConfig
        if max_wall_clock_time:
            raise B2SError("mcts_eval: max_wall_clock_time is not supported (the caller drives the rounds and owns the time budget)")
        self._h = C.c_void_p()
        self.n = roots_batch.n if n_trees is None else int(n_trees)
        self.info = roots_batch.info
        self._dev = roots_batch._dev
        self.leaves = leaves if leaves is not None else BatchedState(roots_batch.game, self.n, roots_batch.device)
        A = self.info.num_distinct_actions
        noise_ptr = None
        if root_noise is not None:
            if root_noise.dtype != torch.float64 or not root_noise.is_cuda or tuple(root_noise.shape) != (self.n, A):
                raise B2SError("mcts_eval: root_noise must be a float64 CUDA tensor of shape [n_trees, num_distinct_actions]")
            root_noise = root_noise.contiguous()
            noise_ptr = root_noise.data_ptr()
        cfg = MctsEvalConfig(int(max_simulations), int(bool(solve)), int(child_selection_policy), 0, float(uct_c), int(seed),
                             int(tree_index_offset), int(max_nodes_total), int(max_nodes_per_tree), float(dirichlet_epsilon),
                             noise_ptr)
        check(lib().b2s_mcts_eval_create(roots_batch._h, self.n, C.byref(cfg), self.leaves._h, C.byref(self._h),
                                         self.leaves._stream()))
        self._pending = torch.zeros((self.n,), dtype=torch.uint8, device=self._dev)

    def __del__(self):
        try:
            if self._h:
                lib().b2s_mcts_eval_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def step(self, values=None, priors=None):
        """One round.  Returns (pending [n] bool tensor, number of pending lanes); 0 pending = the search is over."""
        ptrs = []
        for name, t, width in (("values", values, self.info.num_players), ("priors", priors, self.info.num_distinct_actions)):
            if t is None:
                ptrs.append(None)
                continue
            if t.dtype != torch.float64 or not t.is_cuda or t.dim() != 2 or t.shape[0] < self.n or t.shape[1] != width:
                raise B2SError("mcts_eval: %s must be a float64 CUDA tensor of shape [n_trees, %d]" % (name, width))
            if not t.is_contiguous():
                raise B2SError("mcts_eval: %s must be contiguous" % name)
            ptrs.append(t.data_ptr())
        n_pending = C.c_int64()
        check(lib().b2s_mcts_eval_step(self._h, ptrs[0], ptrs[1], self._pending.data_ptr(), C.byref(n_pending), self.leaves._stream()))
        return self._pending.bool(), n_pending.value

    def results(self):
        """The root statistics so far, as mcts_search returns them (visits, total_reward, outcome_p0, best_action, sims_run,
        gc_runs), plus prior_requests [n] int32: prior-only requests (expansions after a garbage collection freed a node's
        children or cached prior)."""
        n, A, dev = self.n, self.info.num_distinct_actions, self._dev
        out = {
            "visits": torch.empty((n, A), dtype=torch.int32, device=dev),
            "total_reward": torch.empty((n, A), dtype=torch.float64, device=dev),
            "outcome_p0": torch.empty((n, A), dtype=torch.float32, device=dev),
            "best_action": torch.empty((n,), dtype=torch.int32, device=dev),
            "sims_run": torch.empty((n,), dtype=torch.int32, device=dev),
            "gc_runs": torch.empty((n,), dtype=torch.int32, device=dev),
            "prior_requests": torch.empty((n,), dtype=torch.int32, device=dev),
        }
        check(lib().b2s_mcts_eval_results(self._h, *[out[k].data_ptr() for k in ("visits", "total_reward", "outcome_p0", "best_action",
                                                                                  "sims_run", "gc_runs", "prior_requests")],
                                          self.leaves._stream()))
        return out


def mcts_search_evaluated(batch, evaluate, max_simulations, uct_c=2.0, solve=True, seed=0, tree_index_offset=0, n_trees=None,
                          child_selection_policy=ChildSelectionPolicy.UCT, max_nodes_per_tree=0, max_nodes_total=0,
                          root_noise=None, dirichlet_epsilon=0.0, leaves=None, max_wall_clock_time=0.0):
    """Batched MCTSBot.mcts_search with a caller-supplied batched evaluator: `evaluate(leaves, pending) -> (values, priors)`
    gets the leaves BatchedState and the pending mask (device tensors) and returns values [n, num_players] and priors
    [n, num_distinct_actions] for the pending lanes (as MCTSEvalSearch.step takes them; other float dtypes are converted).
    Runs the rounds until every tree has finished and returns MCTSEvalSearch.results() plus "rounds" (evaluate calls) and
    "failed_trees" (trees that stopped because their node arena was full)."""
    search = MCTSEvalSearch(batch, max_simulations, uct_c, solve, seed, tree_index_offset, n_trees, child_selection_policy,
                            max_nodes_per_tree, max_nodes_total, root_noise, dirichlet_epsilon, leaves, max_wall_clock_time)
    values = priors = None
    rounds = 0
    while True:
        pending, n_pending = search.step(values, priors)
        if n_pending == 0:
            break
        rounds += 1
        values, priors = evaluate(search.leaves, pending)
        values = values.to(torch.float64).contiguous()
        priors = priors.to(torch.float64).contiguous()
    out = search.results()
    out["rounds"] = rounds
    out["failed_trees"] = search.leaves.error_count()[0]    # trees that ran out of arena nodes (b2s_error_count)
    return out


class AlphaBetaEvalSearch:
    """algorithms::AlphaBetaSearch (algorithms/minimax.cc:49-137, 221-258) with a caller-supplied value function over n roots
    at once, driven in rounds (b2s_alpha_beta_eval_*): every step() advances all live roots until each needs one value or
    finishes; the states to evaluate are lanes of `.leaves` (a BatchedState of the roots' game), flagged by the returned
    `pending` mask.  The next step() takes their values: a float64 device tensor [n, num_players] whose column maxp is the
    reference's value_function(state), the value of the maximizing player (the shape mcts_search_evaluated's values have).
    step(None) starts the search.  The evaluated states and their order are the reference's value_function calls; terminal
    states are never evaluated.  depth_limit -1 is unlimited, maximizing_player -1 the root's mover, max_nodes 0 no budget."""

    def __init__(self, roots_batch, depth_limit, maximizing_player=-1, max_nodes=0, n=None, leaves=None):
        from ._lib import AlphaBetaConfig
        self._h = C.c_void_p()
        self.n = roots_batch.n if n is None else int(n)
        self.info = roots_batch.info
        self._dev = roots_batch._dev
        self.leaves = leaves if leaves is not None else BatchedState(roots_batch.game, self.n, roots_batch.device)
        cfg = AlphaBetaConfig(int(depth_limit), int(maximizing_player), int(max_nodes))
        check(lib().b2s_alpha_beta_eval_create(roots_batch._h, self.n, C.byref(cfg), self.leaves._h, C.byref(self._h),
                                               self.leaves._stream()))
        self._pending = torch.zeros((self.n,), dtype=torch.uint8, device=self._dev)

    def __del__(self):
        try:
            if self._h:
                lib().b2s_alpha_beta_eval_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def step(self, values=None):
        """One round.  Returns (pending [n] bool tensor, number of pending lanes); 0 pending = the search is over."""
        ptr = None
        if values is not None:
            width = self.info.num_players
            if values.dtype != torch.float64 or not values.is_cuda or values.dim() != 2 or values.shape[0] < self.n or \
                    values.shape[1] != width:
                raise B2SError("alpha_beta_eval: values must be a float64 CUDA tensor of shape [n, %d]" % width)
            if not values.is_contiguous():
                raise B2SError("alpha_beta_eval: values must be contiguous")
            ptr = values.data_ptr()
        n_pending = C.c_int64()
        check(lib().b2s_alpha_beta_eval_step(self._h, ptr, self._pending.data_ptr(), C.byref(n_pending), self.leaves._stream()))
        return self._pending.bool(), n_pending.value

    def results(self):
        """dict of device tensors [n]: value float64, best_action int32 (-1 for a terminal root or a depth-0 root), nodes int64
        (child states generated), status uint8 (0 solved, 1 max_nodes ran out, 3 maximizing_player -1 on a terminal root) and
        evaluations int64 (value-function calls).  Final once step() has reported 0 pending."""
        n, dev = self.n, self._dev
        out = {
            "value": torch.empty((n,), dtype=torch.float64, device=dev),
            "best_action": torch.empty((n,), dtype=torch.int32, device=dev),
            "nodes": torch.empty((n,), dtype=torch.int64, device=dev),
            "status": torch.empty((n,), dtype=torch.uint8, device=dev),
            "evaluations": torch.empty((n,), dtype=torch.int64, device=dev),
        }
        check(lib().b2s_alpha_beta_eval_results(self._h, *[out[k].data_ptr() for k in ("value", "best_action", "nodes", "status",
                                                                                        "evaluations")], self.leaves._stream()))
        return out


def alpha_beta_search_evaluated(batch, value_function, depth_limit, maximizing_player=-1, max_nodes=0, n=None, leaves=None):
    """Batched AlphaBetaSearch with a caller-supplied batched value function: `value_function(leaves, pending)` gets the leaves
    BatchedState and the pending mask (device tensors) and returns values [n, num_players] for the pending lanes (column maxp
    is the maximizing player's value; other float dtypes are converted).  Runs the rounds until every root has finished and
    returns AlphaBetaEvalSearch.results() plus "rounds" (value_function calls)."""
    search = AlphaBetaEvalSearch(batch, depth_limit, maximizing_player, max_nodes, n, leaves)
    values = None
    rounds = 0
    while True:
        pending, n_pending = search.step(values)
        if n_pending == 0:
            break
        rounds += 1
        values = value_function(search.leaves, pending).to(torch.float64).contiguous()
    out = search.results()
    out["rounds"] = rounds
    return out


def dirichlet_noise(batch, alpha, generator=None, n=None):
    """Per lane a Dirichlet(alpha) vector over the lane's legal actions, scattered by action id ([n, A] float64, zero on illegal
    actions): the noise dirichlet_noise (algorithms/mcts.cc:188-203) draws for the root, here drawn in torch as normalised
    Gamma(alpha, 1) variates (torch's own stream, optionally `generator`)."""
    mask = batch.legal_actions_mask(n=n).to(torch.float64)
    conc = torch.full(mask.shape, float(alpha), dtype=torch.float64, device=mask.device)
    g = torch._standard_gamma(conc, generator=generator) * mask
    return g / g.sum(dim=1, keepdim=True).clamp_min(torch.finfo(torch.float64).tiny)


def bind_host_to_device(device=0):
    """Pins the calling thread to the CPUs of the GPU's NUMA node (b2s_bind_host_to_device); returns the CPU count,
    or 0 when the topology cannot be read (containers without sysfs PCI entries)."""
    n = C.c_int(0)
    if lib().b2s_bind_host_to_device(int(device), C.byref(n)) != 0:
        return 0
    return n.value


def mcts_nodes_used(batch):
    v = C.c_int64()
    check(lib().b2s_mcts_nodes_used(batch._h, C.byref(v)))
    return v.value


class RandomRolloutEvaluator:
    """Mirror of algorithms::RandomRolloutEvaluator(n_rollouts, seed) (mcts.h:97-111): a parameter holder; the
    rollouts themselves run inside the device search."""

    def __init__(self, n_rollouts=1, seed=0):
        self.n_rollouts, self.seed = int(n_rollouts), int(seed)


class MCTSBot:
    """Mirror of pyspiel.MCTSBot(game, evaluator, uct_c, max_simulations, max_memory_mb, solve, seed, verbose,
    child_selection_policy) (python/pybind11/bots.cc:129-149, algorithms/mcts.h:161-169) over the device search."""

    def __init__(self, game, evaluator, uct_c, max_simulations, max_memory_mb=1000, solve=True, seed=0, verbose=False,
                 child_selection_policy=ChildSelectionPolicy.UCT):
        if not isinstance(evaluator, RandomRolloutEvaluator):
            raise B2SError("the device MCTSBot supports RandomRolloutEvaluator only")
        self.game, self.evaluator = game, evaluator
        self.uct_c, self.max_simulations, self.solve, self.seed = float(uct_c), int(max_simulations), bool(solve), int(seed)
        # MCTSBot::max_nodes_ = (max_memory_mb << 20) / sizeof(SearchNode) + 1, sizeof(SearchNode) = 80 (mcts.cc:214)
        self.max_nodes = ((int(max_memory_mb) << 20) // 80 + 1) if max_memory_mb else 0
        self.child_selection_policy = int(child_selection_policy)
        self._searches = 0

    def mcts_search(self, state):
        """Returns the root statistics of one search from `state` (a scalar State adapter).  Every search uses a fresh
        random stream (seed, tree index = number of earlier searches), like the reference bot's advancing rng_."""
        self._searches += 1
        return mcts_search(state._b, self.max_simulations, self.uct_c, self.evaluator.n_rollouts, self.solve, self.seed,
                           tree_index_offset=self._searches - 1, n_trees=1, max_nodes_per_tree=self.max_nodes,
                           child_selection_policy=self.child_selection_policy)

    def step(self, state):
        """Bot::Step (mcts.cc:233-266): the best action at `state`."""
        return int(self.mcts_search(state)["best_action"].item())


class CFRSolver:
    """Mirror of pyspiel.CFRSolver(game) (python/pybind11/policy.cc:224-245; algorithms/cfr.h:312-328) with
    device-resident tables.  CFRPlusSolver = CFRSolver(game, linear_averaging=True, regret_matching_plus=True)."""

    def __init__(self, game, linear_averaging=False, regret_matching_plus=False, _mccfr_tables=False, _best_response_opponents=False,
                 _dcfr=None):
        from ._lib import CfrInfo
        if not torch.cuda.is_available():
            raise B2SError("no CUDA device: open_spiel_b200 has no CPU fallback")
        self.game = game
        self._h = C.c_void_p()
        flags = ((1 if linear_averaging else 0) | (2 if regret_matching_plus else 0) | (4 if _mccfr_tables else 0)
                 | (8 if _best_response_opponents else 0))
        self._plus = bool(linear_averaging and regret_matching_plus)
        if _dcfr is None:
            check(lib().b2s_cfr_create(game._gid, C.byref(game._cparams), flags, game.device, C.byref(self._h)))
        else:                   # (alpha, beta, gamma) of a DCFRSolver
            check(lib().b2s_dcfr_create(game._gid, C.byref(game._cparams), *[float(x) for x in _dcfr], game.device,
                                        C.byref(self._h)))
        self._info = CfrInfo()
        check(lib().b2s_cfr_info_get(self._h, C.byref(self._info)))

    def __del__(self):
        try:
            if self._h:
                lib().b2s_cfr_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def info(self):
        from ._lib import CfrInfo
        i = CfrInfo()
        check(lib().b2s_cfr_info_get(self._h, C.byref(i)))
        return i

    def _stream(self):
        """torch's current stream on the solver's device: every call below is ordered on it, as torch's own work is."""
        return C.c_void_p(torch.cuda.current_stream(torch.device("cuda", self.game.device)).cuda_stream)

    def evaluate_and_update_policy(self, iterations=1):
        """CFRSolverBase::EvaluateAndUpdatePolicy (cfr.cc:263-282), `iterations` times in one kernel launch."""
        check(lib().b2s_cfr_iterate(self._h, int(iterations), self._stream()))

    def table(self):
        """The info-state table as numpy arrays: dict(regrets, cum_policy, cur_policy, offsets, legal_actions,
        players, keys) — see b2s_cfr_export."""
        i = self._info
        E, I, T = i.num_entries, i.num_infosets, i.key_floats
        out = {"regrets": np.empty(E), "cum_policy": np.empty(E), "cur_policy": np.empty(E),
               "offsets": np.empty(I + 1, dtype=np.int32), "legal_actions": np.empty(E, dtype=np.int32),
               "players": np.empty(I, dtype=np.int32), "keys": np.empty((I, T), dtype=np.float32)}
        p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
        check(lib().b2s_cfr_export(self._h, p(out["regrets"]), p(out["cum_policy"]), p(out["cur_policy"]),
                                   p(out["offsets"]), p(out["legal_actions"]), p(out["players"]), p(out["keys"]), self._stream()))
        return out

    def load_table(self, regrets=None, cum_policy=None, cur_policy=None, iteration=-1):
        p = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.c_void_p)   # noqa: E731
        keep = [np.ascontiguousarray(a, dtype=np.float64) if a is not None else None for a in (regrets, cum_policy, cur_policy)]
        check(lib().b2s_cfr_import(self._h, *[None if a is None else a.ctypes.data_as(C.c_void_p) for a in keep],
                                   int(iteration), self._stream()))

    def table_pointers(self):
        r, c, u = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(lib().b2s_cfr_tables(self._h, C.byref(r), C.byref(c), C.byref(u)))
        return r.value, c.value, u.value

    def serialize(self, delimiter="<~>"):
        """CFRSolverBase::Serialize (cfr.cc:284-307) with double_precision = -1: text the reference's DeserializeCFRSolver /
        DeserializeCFRPlusSolver loads (information states keyed by their strings, doubles as lossless hex floats)."""
        from . import serialization as ser
        t = self.table()
        i = self.info()
        kind = self._solver_type or ("CFRPlusSolver" if getattr(self, "_plus", False) else "CFRSolver")
        return ser.serialize_cfr_solver(str(self.game), kind, i.iteration, ser.table_keys(self.game._name, t), t, delimiter)

    def load_serialized(self, text, delimiter="<~>"):
        """Load tables and iteration counter from a CFRSolverBase::Serialize text (ours or the reference's)."""
        from . import serialization as ser
        parsed = ser.deserialize_cfr_solver(text, delimiter)
        t = self.table()
        r, c, p = ser.table_arrays_from(parsed["table"], ser.table_keys(self.game._name, t), t)
        self.load_table(r, c, p, iteration=parsed["iteration"])
        return parsed

    _has_current_policy = True
    _solver_type = None         # the [SolverType] serialize() writes, when the flags alone do not name it

    def _require_current_policy(self):
        if not self._has_current_policy:
            raise B2SError("%s keeps no current policy: use the average policy" % type(self).__name__)

    def nash_conv(self, average=True):
        """algorithms::NashConv (tabular_exploitability.cc) of the average (default) or current policy, on the device."""
        if not average:
            self._require_current_policy()
        nc = C.c_double()
        vals = (C.c_double * 4)()
        check(lib().b2s_cfr_nash_conv(self._h, int(bool(average)), C.byref(nc), vals, self._stream()))
        self.last_values = list(vals)
        return nc.value

    def best_response(self, average=True):
        """TabularBestResponse of each player against the other's average (default) / current policy, on the device:
        (actions, values) with actions[I] = the legal action chosen at information state I (table() order; first maximum, as
        best_response.cc:194-228) and values = [BR value p0, BR value p1, on-policy value p0, on-policy value p1]."""
        if not average:
            self._require_current_policy()
        i = self._info
        idx = np.empty(i.num_infosets, dtype=np.int32)
        vals = (C.c_double * 4)()
        check(lib().b2s_cfr_best_response(self._h, int(bool(average)), idx.ctypes.data_as(C.c_void_p), vals, self._stream()))
        t = self.table()
        return t["legal_actions"][t["offsets"][:-1] + idx], list(vals)

    def exploitability(self, average=True):
        """algorithms::Exploitability = NashConv / num_players."""
        return self.nash_conv(average) / 2.0

    def current_policy(self):
        """CFRCurrentPolicy (cfr.cc:139-165): {key bytes: [(action, prob)]} from the current-policy table."""
        self._require_current_policy()
        t = self.table()
        return {t["keys"][k].tobytes(): list(zip(t["legal_actions"][t["offsets"][k]:t["offsets"][k + 1]].tolist(),
                                                 t["cur_policy"][t["offsets"][k]:t["offsets"][k + 1]].tolist()))
                for k in range(len(t["players"]))}

    def tabular_current_policy(self):
        """{information state string: [(action, prob)]} of the current policy."""
        from . import serialization as ser
        t = self.table()
        keys = ser.table_keys(self.game._name, t)
        return {keys[k]: v for k, v in enumerate(self.current_policy().values())}

    def tabular_average_policy(self):
        """pyspiel CFRSolver.tabular_average_policy (python/pybind11/policy.cc:224-245): {information state string:
        [(action, prob)]} — the keys the reference's TabularPolicy uses."""
        from . import serialization as ser
        t = self.table()
        keys = ser.table_keys(self.game._name, t)
        return {keys[k]: v for k, v in enumerate(self.average_policy().values())}

    def average_policy(self):
        """CFRAveragePolicy (cfr.cc:104-125): {key bytes: [(action, prob)]}, uniform where nothing accumulated."""
        t = self.table()
        pol = {}
        for k in range(len(t["players"])):
            lo, hi = t["offsets"][k], t["offsets"][k + 1]
            cp = t["cum_policy"][lo:hi]
            s = 0.0
            for v in cp:
                s += v
            probs = [1.0 / (hi - lo)] * (hi - lo) if s == 0.0 else [v / s for v in cp]
            pol[t["keys"][k].tobytes()] = list(zip(t["legal_actions"][lo:hi].tolist(), probs))
        return pol


class CFRBRSolver(CFRSolver):
    """Mirror of pyspiel.CFRBRSolver(game) (python/pybind11/policy.cc:264-280; algorithms/cfr_br.h) with device-resident
    tables: each iteration both players' pure best responses to the current policy (the uniform policy on iteration 1), then
    each player's traversal against the other's best response, then regret matching.  Tables match the reference bit for
    bit; see B2S_CFR_BEST_RESPONSE_OPPONENTS in include/b2s.h."""

    _solver_type = "CFRBRSolver"

    def __init__(self, game):
        super().__init__(game, _best_response_opponents=True)

    def evaluate_and_update_policy(self, iterations=1):
        """CFRBRSolver::EvaluateAndUpdatePolicy (cfr_br.cc:50-82), `iterations` times in one kernel launch."""
        super().evaluate_and_update_policy(iterations)

    def load_serialized(self, text, delimiter="<~>"):
        """Load a CFRBRSolver Serialize text (ours or the reference's), as DeserializeCFRBRSolver (cfr_br.cc:84-96)."""
        from . import serialization as ser
        kind = ser.deserialize_cfr_solver(text, delimiter)["solver_type"]
        if kind != "CFRBRSolver":
            raise B2SError("CFRBRSolver.load_serialized: the text holds a %r, not a CFRBRSolver" % kind)
        return super().load_serialized(text, delimiter)


class DCFRSolver(CFRSolver):
    """Mirror of python/algorithms/discounted_cfr.py DCFRSolver(game, alpha=3/2, beta=0, gamma=2) with device-resident
    tables (k_dcfr): alternating updates; per iteration t and player, the traversal with average-policy increments
    (reach * pi) * t**gamma, then the player's regrets multiplied by t**alpha / (t**alpha + 1) where >= 0 and by
    t**beta / (t**beta + 1) elsewhere, then regret matching.  Tables match the reference bit for bit; see b2s_dcfr_create
    in include/b2s.h.  average_policy() is cfr.py's _update_average_policy, which is CFRAveragePolicy's rule."""

    def __init__(self, game, alpha=3 / 2, beta=0, gamma=2):
        self.alpha, self.beta, self.gamma = alpha, beta, gamma
        super().__init__(game, _dcfr=(alpha, beta, gamma))

    def evaluate_and_update_policy(self, iterations=1):
        """_DCFRSolver.evaluate_and_update_policy (discounted_cfr.py:190-209), `iterations` times in one kernel launch."""
        super().evaluate_and_update_policy(iterations)

    _NO_TEXT = "%s.%s: no text format: the reference's DCFR has none, and CFRSolver text would resume as plain CFR"

    def serialize(self, delimiter="<~>"):
        raise B2SError(self._NO_TEXT % (type(self).__name__, "serialize"))

    def load_serialized(self, text, delimiter="<~>"):
        raise B2SError(self._NO_TEXT % (type(self).__name__, "load_serialized"))


class LCFRSolver(DCFRSolver):
    """Mirror of python/algorithms/discounted_cfr.py LCFRSolver(game): DCFRSolver with alpha = beta = gamma = 1."""

    def __init__(self, game):
        super().__init__(game, alpha=1, beta=1, gamma=1)


class ExternalSamplingMCCFRSolver(CFRSolver):
    """Mirror of pyspiel.ExternalSamplingMCCFRSolver(game, seed, avg_type=kSimple)
    (algorithms/external_sampling_mccfr.h:55-110) with device-resident tables.  `traversals_per_update` independent
    traversals run in parallel per (iteration, traverser) phase against frozen tables; 1 = the reference's algorithm.
    Like the reference, it has no current policy: simple averaging runs regret matching on a copy and never writes the
    current-policy table, so nash_conv / best_response(average=False) and current_policy() raise B2SError."""

    _has_current_policy = False

    def __init__(self, game, seed=0, traversals_per_update=1, full_average=False):
        """full_average = AverageType::kFull (external_sampling_mccfr.h:53-54) instead of the default kSimple."""
        super().__init__(game, _mccfr_tables=True)
        self.seed, self.traversals_per_update, self.full_average = int(seed), int(traversals_per_update), bool(full_average)

    def run_iteration(self, iterations=1):
        """ExternalSamplingMCCFRSolver::RunIteration (external_sampling_mccfr.cc:71-80), `iterations` times."""
        check(lib().b2s_mccfr_external_iterate_ex(self._h, int(iterations), self.traversals_per_update, self.seed,
                                                  1 if self.full_average else 0, self._stream()))

    def evaluate_and_update_policy(self, iterations=1):
        raise B2SError("ExternalSamplingMCCFRSolver: use run_iteration()")


class OutcomeSamplingMCCFRSolver(CFRSolver):
    """Mirror of pyspiel.OutcomeSamplingMCCFRSolver(game, epsilon, seed) (algorithms/outcome_sampling_mccfr.h:40-66; default
    uniform policy, no baseline) with device-resident tables.  `trajectories_per_update` independent episodes run in parallel
    per (iteration, player) phase against frozen tables; 1 = the reference's algorithm.  No current policy, as for
    ExternalSamplingMCCFRSolver."""

    _has_current_policy = False

    def __init__(self, game, epsilon=0.6, seed=0, trajectories_per_update=1):
        super().__init__(game, _mccfr_tables=True)
        self.epsilon, self.seed, self.trajectories_per_update = float(epsilon), int(seed), int(trajectories_per_update)

    def run_iteration(self, iterations=1):
        """OutcomeSamplingMCCFRSolver::RunIteration (outcome_sampling_mccfr.cc:60-67), `iterations` times."""
        check(lib().b2s_mccfr_outcome_iterate(self._h, int(iterations), self.trajectories_per_update, self.seed, self.epsilon, self._stream()))

    def evaluate_and_update_policy(self, iterations=1):
        raise B2SError("OutcomeSamplingMCCFRSolver: use run_iteration()")

