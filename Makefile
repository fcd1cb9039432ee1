# Builds libkgpu.so (the product: sm_90a kernels for the H100 + C ABI) and the CPU
# oracle (test infrastructure).  `python -c "import __graft_entry__ as g; g.build()"`
# runs exactly this.
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
EXTRA ?=
NVCCFLAGS ?= $(EXTRA) -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wextra -Xptxas -v
CSRC := kubegpu_b200/csrc
LIB := kubegpu_b200/lib/libkgpu.so

HOSTLIB := kubegpu_b200/lib/libkgpu_host.so
CLI := kubegpu_b200/lib/kgpu_sched_cli
CXX ?= g++
CXXFLAGS ?= -O2 -std=c++17 -fPIC -Wall -Wextra

all: $(LIB) $(HOSTLIB) $(CLI) oracle

# C++ mirror of the reference's DeviceScheduler plugin (host layer above the C ABI)
$(HOSTLIB): $(CSRC)/host/device_scheduler.cc $(CSRC)/host/gpus_info.cc $(CSRC)/host/device_scheduler.h $(CSRC)/host/gpus_info.h include/kgpu.h $(LIB)
	$(CXX) $(CXXFLAGS) -shared -o $@ $(CSRC)/host/device_scheduler.cc $(CSRC)/host/gpus_info.cc -Lkubegpu_b200/lib -lkgpu -Wl,-rpath,'$$ORIGIN'

$(CLI): $(CSRC)/host/sched_cli.cc $(HOSTLIB)
	$(CXX) $(CXXFLAGS) -o $@ $(CSRC)/host/sched_cli.cc -Lkubegpu_b200/lib -lkgpu_host -lkgpu -Wl,-rpath,'$$ORIGIN'

$(LIB): $(CSRC)/kgpu.cu $(CSRC)/buffer.h $(CSRC)/score_pairs.cuh $(CSRC)/place_sequential.cuh $(CSRC)/gang_domain.cuh $(CSRC)/preempt.cuh $(CSRC)/preempt_plan.cuh $(CSRC)/preempt_plan_domain.cuh $(CSRC)/score_pairs_sparse.cuh $(CSRC)/sparse_work.h $(CSRC)/launch_plan.h $(CSRC)/peer_exchange.cuh $(CSRC)/node_state.cuh $(CSRC)/subset_dp_sparse_gen.cuh $(CSRC)/subset_dp_gen.cuh $(CSRC)/multi_device.cc $(CSRC)/multi_device.h include/kgpu.h
	@mkdir -p kubegpu_b200/lib
	$(NVCC) $(NVCCFLAGS) -shared -o $@ $(CSRC)/kgpu.cu $(CSRC)/multi_device.cc -ldl

oracle:
	$(MAKE) -s -C oracle

clean:
	rm -rf kubegpu_b200/lib oracle/_build

.PHONY: all oracle clean
