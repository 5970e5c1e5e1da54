"""Regenerates tests/golden/env_reference.json: sha256 digests of every output of the env_lib runs that
tests/test_env_reference.py compares call by call with the reference's own rl_environment.Environment / SyncVectorEnv,
so env_lib stays pinned where no reference checkout exists.  Run after that test passes against the checkout:

  python tests/golden/make_env_reference.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import env_lib  # noqa: E402


def main():
    out = {}
    for gs, kind, rid in env_lib.reference_cases():
        ve = env_lib.VectorEnv(gs, env_lib.REFERENCE_N, env_lib.REFERENCE_SEED, 0, kind)
        out[env_lib.case_id((gs, kind, rid))] = env_lib.digest(env_lib.run_calls(
            ve.reset, ve.step, env_lib.REFERENCE_N, env_lib.REFERENCE_STEPS, env_lib.REFERENCE_SEED, rid))
    with open(os.path.join(HERE, "env_reference.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
