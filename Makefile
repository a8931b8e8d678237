# Builds, in-tree: libmrq.so (the C-ABI engine, sm_90a only), libraftpipe.so (the C++ host side above the
# C-ABI: channels, host node, WAL, NewRaftPipe), the CPU oracle (test infrastructure) and the C++ scenario test.
NVCC ?= /usr/local/cuda/bin/nvcc
CXX ?= g++
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wextra -Xptxas -v
CXXFLAGS := -O2 -std=c++17 -fPIC -Wall -Wextra -pthread
ROOT := $(abspath .)
LIB := raftsql_b200/libmrq.so
HOSTLIB := raftsql_b200/libraftpipe.so
SRC := raftsql_b200/csrc/mrq_engine.cu raftsql_b200/csrc/mrq_pack8_rows.cpp
HDR := raftsql_b200/csrc/mrq_kernels.cuh include/mrq.h include/mrq_trace.h include/mrq_packed8.h
HOSTSRC := raftsql_b200/csrc/host/hostnode.cpp raftsql_b200/csrc/host/raftpipe.cpp
HOSTHDR := raftsql_b200/csrc/host/chan.hpp raftsql_b200/csrc/host/hostnode.hpp raftsql_b200/csrc/host/raftpipe.hpp include/mrq.h
CPPTEST := tests/cpp/raftpipe_test

all: $(LIB) $(HOSTLIB) oracle $(CPPTEST)

$(LIB): $(SRC) $(HDR)
	$(NVCC) $(NVFLAGS) -shared -o $@ $(SRC) -ldl 2> build_ptxas.log || (cat build_ptxas.log; exit 1)

$(HOSTLIB): $(HOSTSRC) $(HOSTHDR) $(LIB)
	$(CXX) $(CXXFLAGS) -shared -o $@ $(HOSTSRC) -L$(ROOT)/raftsql_b200 -lmrq -Wl,-rpath,'$$ORIGIN'

oracle:
	$(MAKE) -C oracle liboracle.so

$(CPPTEST): tests/cpp/raftpipe_test.cpp $(HOSTLIB) oracle
	$(CXX) $(CXXFLAGS) -o $@ tests/cpp/raftpipe_test.cpp -L$(ROOT)/raftsql_b200 -lraftpipe -lmrq -L$(ROOT)/oracle -loracle \
	  -Wl,-rpath,$(ROOT)/raftsql_b200 -Wl,-rpath,$(ROOT)/oracle

# The C++ host side and its scenario test under the sanitizers (CPU suite; oracle core only — no device code runs).
# SAN_CXX: the first of $(CXX), g++, /usr/bin/g++ that ships the sanitizer runtimes (`make san_cxx` prints it).
SAN_CXX := $(shell for c in $(CXX) g++ /usr/bin/g++; do f=`$$c -print-file-name=libtsan.so 2>/dev/null`; \
	if [ -n "$$f" ] && [ "$$f" != libtsan.so ]; then echo $$c; break; fi; done)
SAN_SRC := tests/cpp/raftpipe_test.cpp $(HOSTSRC) oracle/raft_oracle.c
san_cxx:
	@echo $(SAN_CXX)
tests/cpp/raftpipe_test_asan: $(SAN_SRC) $(HOSTHDR) $(LIB)
	$(SAN_CXX) -O1 -g -std=c++17 -pthread -fsanitize=address,undefined -fno-sanitize-recover=undefined -o $@ $(SAN_SRC) \
	  -L$(ROOT)/raftsql_b200 -lmrq -Wl,-rpath,$(ROOT)/raftsql_b200
tests/cpp/raftpipe_test_tsan: $(SAN_SRC) $(HOSTHDR) $(LIB)
	$(SAN_CXX) -O1 -g -std=c++17 -pthread -fsanitize=thread -o $@ $(SAN_SRC) \
	  -L$(ROOT)/raftsql_b200 -lmrq -Wl,-rpath,$(ROOT)/raftsql_b200

# The per-group tick functions of mrq_kernels.cuh compiled for the HOST and run against the oracle (CPU suite):
# the device arithmetic, same source, checked where there is no GPU.  The _san build adds ASan + UBSan.
CUDA_INC ?= /usr/local/cuda/include
TICKHOST_SRC := tests/cpp/tick_host_test.cpp oracle/raft_oracle.c
TICKHOST_DEP := $(TICKHOST_SRC) tests/cpp/device_on_host.hpp oracle/raft_oracle.h $(HDR)
tests/cpp/tick_host_test: $(TICKHOST_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(TICKHOST_SRC)
tests/cpp/tick_host_test_san: $(TICKHOST_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(TICKHOST_SRC)
# The same at the library's 16-bit offset width (it includes tick_host_test.cpp for the harness).
TICKHOST16_SRC := tests/cpp/tick_host16_test.cpp oracle/raft_oracle.c
TICKHOST16_DEP := $(TICKHOST16_SRC) $(TICKHOST_DEP)
tests/cpp/tick_host16_test: $(TICKHOST16_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(TICKHOST16_SRC)
tests/cpp/tick_host16_test_san: $(TICKHOST16_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(TICKHOST16_SRC)
# The library's form: 16-bit offsets and clock-relative leader timers (it includes tick_host_test.cpp for the harness).
TICKCLOCK_SRC := tests/cpp/tick_clock_host_test.cpp oracle/raft_oracle.c
TICKCLOCK_DEP := $(TICKCLOCK_SRC) $(TICKHOST_DEP)
tests/cpp/tick_clock_host_test: $(TICKCLOCK_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(TICKCLOCK_SRC)
tests/cpp/tick_clock_host_test_san: $(TICKCLOCK_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(TICKCLOCK_SRC)
# compact_hot_pair (the quad kernel's two-groups-in-16-bit-lanes hot step) against two scalar hot steps.
TICKPAIR_DEP := tests/cpp/tick_pair_host_test.cpp tests/cpp/device_on_host.hpp $(HDR)
tests/cpp/tick_pair_host_test: $(TICKPAIR_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -o $@ tests/cpp/tick_pair_host_test.cpp
tests/cpp/tick_pair_host_test_san: $(TICKPAIR_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -o $@ tests/cpp/tick_pair_host_test.cpp
# Every case of tick_clock_host_test with the quad kernel's pair structure (it includes tick_clock_host_test.cpp).
TICKPAIRCLOCK_SRC := tests/cpp/tick_pair_clock_host_test.cpp oracle/raft_oracle.c
TICKPAIRCLOCK_DEP := $(TICKPAIRCLOCK_SRC) $(TICKCLOCK_DEP)
tests/cpp/tick_pair_clock_host_test: $(TICKPAIRCLOCK_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(TICKPAIRCLOCK_SRC)
tests/cpp/tick_pair_clock_host_test_san: $(TICKPAIRCLOCK_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(TICKPAIRCLOCK_SRC)

# The change feed: the general tick's records against the diff of consecutive oracle exports, and the fast functions
# leaving term / vote / role / lead alone (it includes tick_host_test.cpp for the harness).
FEEDHOST_SRC := tests/cpp/change_feed_host_test.cpp oracle/raft_oracle.c
FEEDHOST_DEP := $(FEEDHOST_SRC) $(TICKHOST_DEP)
tests/cpp/change_feed_host_test: $(FEEDHOST_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(FEEDHOST_SRC)
tests/cpp/change_feed_host_test_san: $(FEEDHOST_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(FEEDHOST_SRC)

# The state of a list of groups: export_group_row / import_group_row over mode-4 states reached by traces and soups,
# against materialise_group and the oracle (it includes tick_host_test.cpp for the harness).
GROUPHOST_SRC := tests/cpp/group_state_host_test.cpp oracle/raft_oracle.c
GROUPHOST_DEP := $(GROUPHOST_SRC) $(TICKHOST_DEP)
tests/cpp/group_state_host_test: $(GROUPHOST_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(GROUPHOST_SRC)
tests/cpp/group_state_host_test_san: $(GROUPHOST_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(GROUPHOST_SRC)

# The fresh groups of mrq_resize_groups: init_state_kernel's rows against create's and the oracle's, for R = 1..8.
RESIZEHOST_SRC := tests/cpp/resize_host_test.cpp oracle/raft_oracle.c
RESIZEHOST_DEP := $(RESIZEHOST_SRC) tests/cpp/device_on_host.hpp oracle/raft_oracle.h $(HDR)
tests/cpp/resize_host_test: $(RESIZEHOST_DEP)
	$(CXX) -std=c++17 -O1 -I$(CUDA_INC) -pthread -o $@ $(RESIZEHOST_SRC)
tests/cpp/resize_host_test_san: $(RESIZEHOST_DEP)
	$(SAN_CXX) -std=c++17 -O0 -fsanitize=address,undefined -fno-sanitize-recover=undefined -I$(CUDA_INC) -pthread -o $@ $(RESIZEHOST_SRC)

clean:
	rm -f $(LIB) $(HOSTLIB) $(CPPTEST) tests/cpp/raftpipe_test_asan tests/cpp/raftpipe_test_tsan build_ptxas.log \
	  tests/cpp/tick_host_test tests/cpp/tick_host_test_san tests/cpp/tick_host16_test tests/cpp/tick_host16_test_san \
	  tests/cpp/tick_clock_host_test tests/cpp/tick_clock_host_test_san tests/cpp/tick_pair_host_test tests/cpp/tick_pair_host_test_san \
	  tests/cpp/tick_pair_clock_host_test tests/cpp/tick_pair_clock_host_test_san \
	  tests/cpp/change_feed_host_test tests/cpp/change_feed_host_test_san tests/cpp/group_state_host_test tests/cpp/group_state_host_test_san \
	  tests/cpp/resize_host_test tests/cpp/resize_host_test_san
	$(MAKE) -C oracle clean
.PHONY: all oracle clean san_cxx
