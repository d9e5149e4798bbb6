# Top-level build: libsalmon_b200.so (CUDA, sm_90a only) + the oracle (test infra).
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xcompiler -Wall -Xcompiler -fopenmp $(PTXAS_V)
CSRC      := salmon_b200/csrc
LIB       := salmon_b200/libsalmon_b200.so
SRCS      := $(wildcard $(CSRC)/*.cu)
HDRS      := $(wildcard $(CSRC)/*.h $(CSRC)/*.cuh include/*.h)

CLI       := salmon_b200/sb_salmon

all: $(LIB) $(CLI) oracle

# one object per translation unit (build/ is git-ignored), so that `make -j` compiles them side by side; the library
# is written under a temporary name and renamed, a snapshot of the tree never sees a half-written .so
OBJS      := $(patsubst $(CSRC)/%.cu,build/%.o,$(SRCS))

build/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -c -o $@ $<

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@.tmp $(OBJS) -ldl -lgomp -lz && mv -f $@.tmp $@

# command-line front end (host C++ over the C ABI; finds the library next to itself)
$(CLI): $(CSRC)/cli_main.cpp $(LIB) include/salmon_b200.h
	g++ -O2 -std=c++17 -Wall -o $@.tmp $(CSRC)/cli_main.cpp -Lsalmon_b200 -lsalmon_b200 -lpthread -Wl,-rpath,'$$ORIGIN' && mv -f $@.tmp $@

oracle:
	$(MAKE) -C oracle

clean:
	rm -rf $(LIB) $(CLI) build; $(MAKE) -C oracle clean

.PHONY: all oracle clean
