# The host program of the affinity flattening in the C++ mirror (kb::actions::allocate::Flatten, FlattenPodAffinity):
# make -C tests/host -f affinity.mk
CXX ?= g++
all: affinity_run
affinity_run: affinity_run.cpp ../../kube_batch_b200/host/kbhost.hpp ../../include/kbgpu.h
	$(CXX) -O1 -std=c++17 -Wall -Wextra -o $@ affinity_run.cpp -L../../kube_batch_b200 -lkbgpu -Wl,-rpath,'$$ORIGIN/../../kube_batch_b200'
.PHONY: all
