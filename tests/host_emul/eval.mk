# TEST INFRASTRUCTURE ONLY: host build of the caller-evaluated MCTS kernel bodies for CPU unit tests (see emul_eval.cc).
CXX := /usr/bin/g++
CUDA_INC ?= /usr/local/cuda/include
libemul_eval.so: emul_eval.cc $(wildcard ../../open_spiel_b200/csrc/rules_*.cuh) ../../open_spiel_b200/csrc/common.cuh ../../open_spiel_b200/csrc/host_compat.h ../../open_spiel_b200/csrc/mcts.cuh ../../open_spiel_b200/csrc/mcts_eval.cuh ../../include/b2s.h
	$(CXX) -std=c++17 -O2 -w -fPIC -shared -I $(CUDA_INC) -o $@ emul_eval.cc
