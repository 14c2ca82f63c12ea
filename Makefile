# Builds the product library (CUDA, sm_90a) and the test oracle (CPU).
#   make            -> xllm_service_b200/libxllm_ingest.so + oracle/liboracle.so
#   make lib | oracle | ref | clean      (ref = oracle/_ref/libxllm_ref.so, the reference's own files; needs the reference checkout, XLLM_REFERENCE_DIR)
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
CC        ?= gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function -Iinclude --expt-relaxed-constexpr
PKG       := xllm_service_b200
CSRC      := $(PKG)/csrc
LIB       := $(PKG)/libxllm_ingest.so
CU_SRCS   := $(wildcard $(CSRC)/*.cu)
CC_SRCS   := $(wildcard $(CSRC)/*.cc)
OBJS      := $(patsubst $(CSRC)/%.cu,build/%.cu.o,$(CU_SRCS)) $(patsubst $(CSRC)/%.cc,build/%.cc.o,$(CC_SRCS))
HDRS      := $(wildcard $(CSRC)/*.h $(CSRC)/*.cuh include/*.h)

ORACLE_LIB  := oracle/liboracle.so
ORACLE_C    := $(wildcard oracle/*.c)
ORACLE_CC   := $(wildcard oracle/*.cc)
ORACLE_OBJS := $(patsubst oracle/%.c,build/oracle/%.c.o,$(ORACLE_C)) $(patsubst oracle/%.cc,build/oracle/%.cc.o,$(ORACLE_CC))

all: lib oracle ref
ref:
	@bash oracle/build_ref.sh
lib: $(LIB)
oracle: $(ORACLE_LIB)

build/%.cu.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -c $< -o $@
build/%.cc.o: $(CSRC)/%.cc $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -x cu -c $< -o $@
$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $^ -lcudart -ldl

build/oracle/%.c.o: oracle/%.c
	@mkdir -p build/oracle
	$(CC) -O3 -march=native -fPIC -Wall -c $< -o $@
build/oracle/%.cc.o: oracle/%.cc $(wildcard oracle/*.h)
	@mkdir -p build/oracle
	$(CXX) -O3 -march=native -std=c++17 -fPIC -Wall -c $< -o $@
$(ORACLE_LIB): $(ORACLE_OBJS)
	$(CXX) -shared -o $@ $^ -lpthread

clean:
	rm -rf build $(LIB) $(ORACLE_LIB)
.PHONY: all lib oracle ref clean
