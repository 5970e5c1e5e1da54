# TEST INFRASTRUCTURE ONLY: host build of the RL environment step's per-lane body for CPU unit tests (see emul_env.cc).
CXX := /usr/bin/g++
CUDA_INC ?= /usr/local/cuda/include
libemul_env.so: emul_env.cc $(wildcard ../../open_spiel_b200/csrc/rules_*.cuh) ../../open_spiel_b200/csrc/common.cuh ../../open_spiel_b200/csrc/env_step.cuh ../../open_spiel_b200/csrc/host_compat.h ../../include/b2s.h
	$(CXX) -std=c++17 -O2 -w -fPIC -shared -I $(CUDA_INC) -o $@ emul_env.cc
