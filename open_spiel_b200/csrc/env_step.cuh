// One RL environment time step of one lane (python/rl_environment.py Environment.step / reset, python/vector_env.py
// SyncVectorEnv.step): the per-lane body of k_env_step (batch_kernels.cuh).  It is also compiled for the host by the CPU
// emulation of the kernel (tests/host_emul/emul_env.cc), so it touches nothing but the lane's state and ctx.
#pragma once
#include "common.cuh"

namespace b2s {

// rl_environment.py StepType
enum EnvStepType : unsigned char { kEnvFirst = 0, kEnvMid = 1, kEnvLast = 2 };

// Random block of the call with counter c: chance node j after the action takes block env_block(c) + 1 + j, chance node j after
// a reset env_block(c) + 32 + j (traj_resolve_chance adds 1 + j).
__host__ __device__ __forceinline__ u32 env_block(unsigned long long c) { return 64u * (u32)(c + 1); }

// Environment.reset (rl_environment.py:399-420): the initial state, its chance nodes resolved (_sample_external_events).
template <class R, class Draw>
__device__ __forceinline__ void env_reset_lane(typename R::S& s, const typename R::Cfg& cfg, const Ctx& ctx, long long i, int mask_words,
                                               Draw& draw, u32 b0) {
  R::init(s, cfg, ctx, i);
  traj_resolve_chance<R>(s, cfg, ctx, i, mask_words, draw, b0 + 31u);
}

// The step of lane i with action a; s holds the lane's state on entry and its new state on return.  Returns the step type and
// writes the rewards r[kPlayers] (State::Rewards(): zero until terminal, then Returns()) and done (the episode ended in this
// step).  `changed` is set when s differs from the entry state (the caller then stores it).
//   reset:                  Environment.reset: every lane starts a new episode, FIRST.
//   s terminal:             Environment.step after LAST (rl_environment.py:372-373): a is ignored, new episode, FIRST.
//   a == -1:                the lane is untouched: MID.
//   otherwise:              apply a (an illegal action is flagged, the lane keeps its state), then resolve chance
//                           (rl_environment.py:375-383): MID, or LAST with done = 1 and the Returns() as rewards.
//   reset_if_done and done: SyncVectorEnv.step(reset_if_done=True) (vector_env.py:54-64): rewards and done of the step are
//                           kept, the lane starts a new episode, FIRST.
template <class R, class Draw>
__device__ __forceinline__ unsigned char env_step_lane(typename R::S& s, int a, bool reset, bool reset_if_done, const typename R::Cfg& cfg,
                                                       const Ctx& ctx, long long i, int mask_words, Draw& draw, u32 b0, float* r,
                                                       unsigned char& done, bool& changed) {
  for (int p = 0; p < R::kPlayers; ++p) r[p] = 0.f;
  done = 0;
  changed = false;
  if (reset || R::terminal(s, cfg)) {
    env_reset_lane<R>(s, cfg, ctx, i, mask_words, draw, b0);
    changed = true;
    return kEnvFirst;
  }
  if (a == -1) return kEnvMid;
  const typename R::S s0 = s;
  if (!R::apply(s, a, cfg, ctx, i)) {
    s = s0;
    flag_error(ctx.err, ctx.lane0 + i);
    return kEnvMid;
  }
  traj_resolve_chance<R>(s, cfg, ctx, i, mask_words, draw, b0);
  changed = true;
  if (!R::terminal(s, cfg)) return kEnvMid;
  R::returns(s, cfg, r);
  done = 1;
  if (!reset_if_done) return kEnvLast;
  env_reset_lane<R>(s, cfg, ctx, i, mask_words, draw, b0);
  return kEnvFirst;
}

}  // namespace b2s
