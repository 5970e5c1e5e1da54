# TEST INFRASTRUCTURE ONLY: host builds of the rule cores and MCTS kernel bodies with go 10..19 (emul_go_wide.cc,
# emul_eval_go_wide.cc) for the CPU tests of tests/test_go_large_*.py.
CXX := /usr/bin/g++
CUDA_INC ?= /usr/local/cuda/include
DEPS := $(wildcard ../../open_spiel_b200/csrc/rules_*.cuh) ../../open_spiel_b200/csrc/common.cuh ../../open_spiel_b200/csrc/host_compat.h \
        ../../open_spiel_b200/csrc/mcts.cuh ../../open_spiel_b200/csrc/mcts_eval.cuh ../../include/b2s.h
all: libemul_go_wide.so libemul_eval_go_wide.so
libemul_go_wide.so: emul_go_wide.cc emul.cc $(DEPS)
	$(CXX) -std=c++17 -O2 -w -fPIC -shared -I $(CUDA_INC) -o $@ emul_go_wide.cc
libemul_eval_go_wide.so: emul_eval_go_wide.cc emul_eval.cc $(DEPS)
	$(CXX) -std=c++17 -O2 -w -fPIC -shared -I $(CUDA_INC) -o $@ emul_eval_go_wide.cc
