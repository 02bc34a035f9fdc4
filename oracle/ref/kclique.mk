# Builds oracle/_ref/ref_kclique_driver: the UNMODIFIED reference CPU app
# kclique (sources under $(REFERENCE)), ref_kclique_driver.cc and the
# functional shims; same flags as core.mk.  Outputs only into oracle/_ref/
# (git-ignored build products).
REFERENCE ?= /root/reference
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -march=x86-64-v3 -fopenmp -pthread -w
INC = -Ishims -I$(REFERENCE) -I$(REFERENCE)/thirdparty -I$(REFERENCE)/examples/analytical_apps
OUT = ../_ref

all: $(OUT)/ref_kclique_driver

$(OUT)/ref_kclique_driver: ref_kclique_driver.cc ../rmat_gen.h shims/mpi.h shims/glog/logging.h
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INC) -include unistd.h ref_kclique_driver.cc $(REFERENCE)/grape/io/local_io_adaptor.cc \
	  $(REFERENCE)/grape/utils/memory_tracker.cc -o $@

.PHONY: all
