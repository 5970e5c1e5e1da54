# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/libspiel_ref_mcts_eval.so: the unmodified reference's MCTSBot driven by the
# deterministic test evaluator (ref_glue/ref_mcts_eval.cc).  It links against _ref/libspiel_ref_c.so from ref_build.mk (run
# that first, with the same REF / JSON_INC), so a process that loads both holds one copy of the reference (one game registry).
#   make -C oracle -f ref_eval.mk REF=<open_spiel checkout> JSON_INC=<dir of nlohmann/json.hpp>
REF ?= $(OPEN_SPIEL_REFERENCE)
CXX := /usr/bin/g++
CXXFLAGS := -std=c++20 -O3 -DNDEBUG -fPIC -w -I absl_shim -I $(REF) $(if $(JSON_INC),-I $(JSON_INC))

_ref/libspiel_ref_mcts_eval.so: ref_glue/ref_mcts_eval.cc _ref/libspiel_ref_c.so
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_glue/ref_mcts_eval.cc -L _ref -l:libspiel_ref_c.so -Wl,-rpath,'$$ORIGIN' -lpthread
