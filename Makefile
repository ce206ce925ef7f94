# Top-level build: the product library, the C host, and (test infrastructure) the oracle.
#
#   make            -> dump1090_b200/libmodes_b200.so + dump1090-b200 (C host)
#   make oracle     -> oracle/_build/libmodes_oracle.so (+ oracle/_ref when /root/reference exists)
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -Iinclude -Xcompiler -fPIC,-Wall,-Wextra
CSRC      := dump1090_b200/csrc
LIB       := dump1090_b200/libmodes_b200.so
OBJS      := build/modes_kernels.o build/modes_scan2.o build/modes_eval_fused.o build/modes_resolve_gpu.o build/modes_api.o build/modes_resolve.o build/modes_tables.o build/modes_format.o build/modes_tracker.o build/modes_pool.o

all: $(LIB) dump1090-b200

build/%.o: $(CSRC)/%.cu $(CSRC)/modes_internal.h $(CSRC)/modes_eval_serial.cuh $(CSRC)/modes_scan_core.cuh $(CSRC)/modes_resolve_core.cuh include/modes_b200.h
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@

build/%.o: $(CSRC)/%.cpp $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -cudart static

dump1090-b200: host/dump1090_b200.c include/modes_b200.h $(LIB)
	gcc -O2 -g -Wall -W -Iinclude -o $@ host/dump1090_b200.c -Ldump1090_b200 -lmodes_b200 -Wl,-rpath,'$$ORIGIN/dump1090_b200' -lm

oracle:
	$(MAKE) -C oracle
	if [ -d /root/reference ]; then $(MAKE) -C oracle ref; fi

# test infrastructure: host build of the per-candidate evaluation (logic checked against the oracle on CPU)
shim: tests/_build/libeval_serial_host.so tests/_build/libscan_core_host.so tests/_build/libresolve_core_host.so
tests/_build/libresolve_core_host.so: tests/host_shim/resolve_core_host.cpp $(CSRC)/modes_resolve_core.cuh include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) tests/host_shim/resolve_core_host.cpp -o $@
tests/_build/libscan_core_host.so: tests/host_shim/scan_core_host.cpp $(CSRC)/modes_scan_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/scan_core_host.cpp -o $@
tests/_build/libeval_serial_host.so: tests/host_shim/eval_serial_host.cpp $(CSRC)/modes_eval_serial.cuh $(CSRC)/modes_tables.cpp include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) -I/usr/local/cuda/include \
	    tests/host_shim/eval_serial_host.cpp $(CSRC)/modes_tables.cpp -o $@

clean:
	rm -rf build tests/_build $(LIB) dump1090-b200

.PHONY: all oracle shim clean
