# The host programs of the action-list mirror (kb::actions::cycle): make -C tests/host -f cycle.mk
CXX ?= g++
all: evict_test cycle_run
evict_test: evict_test.cpp ../../kube_batch_b200/host/kbhost.hpp ../../include/kbgpu.h
	$(CXX) -O1 -std=c++17 -Wall -Wextra -o $@ evict_test.cpp -L../../kube_batch_b200 -lkbgpu -Wl,-rpath,'$$ORIGIN/../../kube_batch_b200'
cycle_run: cycle_run.cpp ../../kube_batch_b200/host/kbhost.hpp ../../include/kbgpu.h
	$(CXX) -O1 -std=c++17 -Wall -Wextra -o $@ cycle_run.cpp -L../../kube_batch_b200 -lkbgpu -Wl,-rpath,'$$ORIGIN/../../kube_batch_b200'
.PHONY: all
