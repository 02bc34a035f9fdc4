# Builds oracle/_ref/ref_pagerank_local_driver: the UNMODIFIED reference CPU app PageRankLocal
# (pagerank/pagerank_local.h, sources under $(REFERENCE)), ref_pagerank_local_driver.cc and the
# functional shims; same flags as Makefile's ref_driver.  Outputs only into oracle/_ref/ (git-ignored
# build products).
REFERENCE ?= /root/reference
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -march=x86-64-v3 -fopenmp -pthread -w
INC = -Ishims -I$(REFERENCE) -I$(REFERENCE)/thirdparty -I$(REFERENCE)/examples/analytical_apps
OUT = ../_ref

all: $(OUT)/ref_pagerank_local_driver

$(OUT)/ref_pagerank_local_driver: ref_pagerank_local_driver.cc ../rmat_gen.h shims/mpi.h shims/glog/logging.h
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INC) -include unistd.h ref_pagerank_local_driver.cc $(REFERENCE)/grape/io/local_io_adaptor.cc \
	  $(REFERENCE)/grape/utils/memory_tracker.cc -o $@

.PHONY: all
