# TEST INFRASTRUCTURE ONLY.  Compiles the UNMODIFIED reference sources of the hot path, from the OpenSpiel source tree
# named by REF (default: $OPEN_SPIEL_REFERENCE), against oracle/absl_shim (abseil is not vendored in the reference).
# Outputs go to oracle/_ref/ only (git-ignored).
#   make -C oracle -f ref_build.mk REF=<open_spiel checkout>   -> _ref/libspiel_ref.a, _ref/ref_bench, _ref/libspiel_ref_c.so
REF ?= $(OPEN_SPIEL_REFERENCE)
CXX := /usr/bin/g++
# Reference Release flags: open_spiel/CMakeLists.txt:56-61 (-O3 -DNDEBUG); C++20 for the shim's std::span-era library.
# JSON_INC: a directory holding nlohmann/json.hpp (the reference clones it; __graft_entry__.json_include_dir() finds one)
CXXFLAGS := -std=c++20 -O3 -DNDEBUG -fPIC -w -I absl_shim -I $(REF) $(if $(JSON_INC),-I $(JSON_INC))
OS := $(REF)/open_spiel
SRCS := spiel.cc spiel_utils.cc game_parameters.cc observer.cc policy.cc spiel_bots.cc simultaneous_move_game.cc \
        action_view.cc utils/status.cc utils/usage_logging.cc \
        games/tic_tac_toe/tic_tac_toe.cc games/connect_four/connect_four.cc games/breakthrough/breakthrough.cc \
        games/hex/hex.cc games/kuhn_poker/kuhn_poker.cc games/leduc_poker/leduc_poker.cc \
        games/go/go.cc games/go/go_board.cc games/mnk/mnk.cc games/othello/othello.cc games/y/y.cc games/havannah/havannah.cc \
        algorithms/mcts.cc algorithms/cfr.cc algorithms/evaluate_bots.cc algorithms/tabular_exploitability.cc \
        algorithms/best_response.cc algorithms/expected_returns.cc algorithms/history_tree.cc \
        algorithms/get_all_states.cc algorithms/trajectories.cc \
        algorithms/external_sampling_mccfr.cc algorithms/outcome_sampling_mccfr.cc tests/basic_tests.cc \
        game_transforms/start_at.cc
OBJS := $(addprefix _ref/obj/,$(SRCS:.cc=.o))

all: _ref/libspiel_ref.a _ref/libspiel_ref_c.so _ref/ref_bench

_ref/obj/%.o: $(OS)/%.cc absl_shim/shim_all.h
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@

_ref/libspiel_ref.a: $(OBJS)
	ar rcs $@ $(OBJS)

# our own glue (NOT reference code): a C ABI over the reference's Game/State/MCTSBot/CFRSolver for tests,
# and the CPU timing harness used by bench.py.
_ref/libspiel_ref_c.so: ref_glue/ref_c_api.cc _ref/libspiel_ref.a
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_glue/ref_c_api.cc -Wl,--whole-archive _ref/libspiel_ref.a -Wl,--no-whole-archive -lpthread

_ref/ref_bench: ref_glue/ref_bench.cc _ref/libspiel_ref.a
	$(CXX) $(CXXFLAGS) -o $@ ref_glue/ref_bench.cc -Wl,--whole-archive _ref/libspiel_ref.a -Wl,--no-whole-archive -lpthread

clean:
	rm -rf _ref
