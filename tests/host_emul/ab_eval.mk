# TEST INFRASTRUCTURE ONLY: host build of the AlphaBetaSearch value-function step kernel for CPU unit tests (see emul_ab_eval.cc).
CXX := /usr/bin/g++
CUDA_INC ?= /usr/local/cuda/include
libemul_ab_eval.so: emul_ab_eval.cc $(wildcard ../../open_spiel_b200/csrc/rules_*.cuh) ../../open_spiel_b200/csrc/common.cuh ../../open_spiel_b200/csrc/alpha_beta.cuh ../../open_spiel_b200/csrc/host_compat.h ../../include/b2s.h
	$(CXX) -std=c++17 -O2 -w -fPIC -shared -I $(CUDA_INC) -o $@ emul_ab_eval.cc
