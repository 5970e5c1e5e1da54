# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/libspiel_ref_cfr_br.so: the UNMODIFIED reference's algorithms/cfr_br.cc
# (CFRBRSolver) with a C ABI over it and over TabularBestResponse (ref_glue/ref_cfr_br.cc).  It links against
# _ref/libspiel_ref_c.so from ref_build.mk (run that first, with the same REF / JSON_INC), which holds the rest of the
# reference, so a process that loads both holds one copy of it (one game registry).
#   make -C oracle -f ref_cfr_br.mk REF=<open_spiel checkout> JSON_INC=<dir of nlohmann/json.hpp>
REF ?= $(OPEN_SPIEL_REFERENCE)
CXX := /usr/bin/g++
CXXFLAGS := -std=c++20 -O3 -DNDEBUG -fPIC -w -I absl_shim -I $(REF) $(if $(JSON_INC),-I $(JSON_INC))

_ref/libspiel_ref_cfr_br.so: ref_glue/ref_cfr_br.cc _ref/cfr_br/cfr_br.o _ref/libspiel_ref_c.so
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_glue/ref_cfr_br.cc _ref/cfr_br/cfr_br.o -L _ref -l:libspiel_ref_c.so -Wl,-rpath,'$$ORIGIN' -lpthread

_ref/cfr_br/cfr_br.o: $(REF)/open_spiel/algorithms/cfr_br.cc absl_shim/shim_all.h
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
