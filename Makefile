# Top-level build: the product library, the C host, and (test infrastructure) the oracle.
#
#   make            -> dump1090_b200/libmodes_b200.so + dump1090-b200 (C host)
#   make oracle     -> oracle/_build/libmodes_oracle.so (+ oracle/_ref when /root/reference exists)
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -Iinclude -Xcompiler -fPIC,-Wall,-Wextra
CSRC      := dump1090_b200/csrc
LIB       := dump1090_b200/libmodes_b200.so
OBJS      := build/modes_kernels.o build/modes_scan2.o build/modes_eval_fused.o build/modes_signal.o build/modes_levels.o build/modes_spectrum.o build/modes_recover.o build/modes_weak.o build/modes_resample.o build/modes_resolve_gpu.o build/modes_api.o build/modes_resolve.o build/modes_tables.o build/modes_format.o build/modes_tracker.o build/modes_pool.o

all: $(LIB) dump1090-b200

build/%.o: $(CSRC)/%.cu $(CSRC)/modes_internal.h $(CSRC)/modes_eval_serial.cuh $(CSRC)/modes_scan_core.cuh $(CSRC)/modes_resolve_core.cuh $(CSRC)/modes_signal_core.cuh $(CSRC)/modes_arrival_core.cuh $(CSRC)/modes_carrier_core.cuh $(CSRC)/modes_levels_core.cuh $(CSRC)/modes_recover_core.cuh $(CSRC)/modes_weak_core.cuh $(CSRC)/modes_resample_core.cuh $(CSRC)/modes_input_core.cuh $(CSRC)/modes_spectrum_core.cuh $(CSRC)/modes_stage.cuh include/modes_b200.h
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@

build/%.o: $(CSRC)/%.cpp $(CSRC)/modes_internal.h $(CSRC)/modes_carrier_core.cuh $(CSRC)/modes_resolve_core.cuh $(CSRC)/modes_input_core.cuh $(CSRC)/modes_resample_core.cuh $(CSRC)/modes_spectrum_core.cuh include/modes_b200.h
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
shim: tests/_build/libeval_serial_host.so tests/_build/libscan_core_host.so tests/_build/libresolve_core_host.so tests/_build/libsignal_core_host.so tests/_build/liblevels_core_host.so tests/_build/librecover_core_host.so tests/_build/libweak_core_host.so tests/_build/libarrival_core_host.so tests/_build/libresample_core_host.so tests/_build/libinput_core_host.so tests/_build/libpool_carry_host.so tests/_build/libdecimate_core_host.so tests/_build/libshift_core_host.so tests/_build/libspectrum_core_host.so tests/_build/libcarrier_core_host.so
tests/_build/libcarrier_core_host.so: tests/host_shim/carrier_core_host.cpp $(CSRC)/modes_carrier_core.cuh $(CSRC)/modes_arrival_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/carrier_core_host.cpp -o $@
tests/_build/libspectrum_core_host.so: tests/host_shim/spectrum_core_host.cpp $(CSRC)/modes_spectrum_core.cuh $(CSRC)/modes_resample_core.cuh include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) tests/host_shim/spectrum_core_host.cpp -o $@
tests/_build/libshift_core_host.so: tests/host_shim/shift_core_host.cpp $(CSRC)/modes_resample_core.cuh $(CSRC)/modes_input_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/shift_core_host.cpp -o $@
tests/_build/libdecimate_core_host.so: tests/host_shim/decimate_core_host.cpp $(CSRC)/modes_resample_core.cuh $(CSRC)/modes_input_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/decimate_core_host.cpp -o $@
tests/_build/libpool_carry_host.so: tests/host_shim/pool_carry_host.cpp $(CSRC)/modes_input_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/pool_carry_host.cpp -o $@
tests/_build/libinput_core_host.so: tests/host_shim/input_core_host.cpp $(CSRC)/modes_input_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/input_core_host.cpp -o $@
tests/_build/libresample_core_host.so: tests/host_shim/resample_core_host.cpp $(CSRC)/modes_resample_core.cuh
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -I$(CSRC) tests/host_shim/resample_core_host.cpp -o $@
tests/_build/libarrival_core_host.so: tests/host_shim/arrival_core_host.cpp $(CSRC)/modes_arrival_core.cuh $(CSRC)/modes_signal_core.cuh $(CSRC)/modes_tables.cpp include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) -I/usr/local/cuda/include \
	    tests/host_shim/arrival_core_host.cpp $(CSRC)/modes_tables.cpp -o $@
tests/_build/libweak_core_host.so: tests/host_shim/weak_core_host.cpp $(CSRC)/modes_weak_core.cuh $(CSRC)/modes_tables.cpp include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) -I/usr/local/cuda/include \
	    tests/host_shim/weak_core_host.cpp $(CSRC)/modes_tables.cpp -o $@
tests/_build/librecover_core_host.so: tests/host_shim/recover_core_host.cpp $(CSRC)/modes_recover_core.cuh $(CSRC)/modes_signal_core.cuh $(CSRC)/modes_tables.cpp include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) -I/usr/local/cuda/include \
	    tests/host_shim/recover_core_host.cpp $(CSRC)/modes_tables.cpp -o $@
tests/_build/liblevels_core_host.so: tests/host_shim/levels_core_host.cpp $(CSRC)/modes_levels_core.cuh $(CSRC)/modes_tables.cpp include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) -I/usr/local/cuda/include \
	    tests/host_shim/levels_core_host.cpp $(CSRC)/modes_tables.cpp -o $@
tests/_build/libsignal_core_host.so: tests/host_shim/signal_core_host.cpp $(CSRC)/modes_signal_core.cuh $(CSRC)/modes_tables.cpp include/modes_b200.h
	@mkdir -p tests/_build
	g++ -O2 -std=c++17 -shared -fPIC -Wall -Wno-unknown-pragmas -x c++ -Iinclude -I$(CSRC) -I/usr/local/cuda/include \
	    tests/host_shim/signal_core_host.cpp $(CSRC)/modes_tables.cpp -o $@
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

# test infrastructure: device harness over the product's own kernel objects (recovery and signal
# passes on constructed corpora, and the exhaustive sweeps of the core headers' device build)
DSHIM_OBJS := build/modes_recover.o build/modes_signal.o build/modes_levels.o build/modes_tables.o
dshim: tests/_build/libkernels_device.so tests/_build/libarrival_device.so tests/_build/libscan_eval_device.so tests/_build/libresample_pool_device.so tests/_build/libresolve_device.so tests/_build/libinput_device.so tests/_build/libconvert_pool_device.so tests/_build/librate_spectrum_device.so tests/_build/libcarrier_device.so tests/_build/libgather_pool_device.so
tests/_build/libkernels_device.so: tests/device_shim/kernels_device.cu $(DSHIM_OBJS) $(CSRC)/modes_internal.h $(CSRC)/modes_signal_core.cuh $(CSRC)/modes_levels_core.cuh include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/kernels_device.cu -o tests/_build/kernels_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/kernels_device.o $(DSHIM_OBJS) -cudart static
# the arrival-time measurement of the signal pass on constructed corpora (tests/test_arrival.py)
tests/_build/libarrival_device.so: tests/device_shim/arrival_device.cu build/modes_signal.o build/modes_tables.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/arrival_device.cu -o tests/_build/arrival_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/arrival_device.o build/modes_signal.o build/modes_tables.o -cudart static
# the carrier measurement of the signal pass on constructed corpora (tests/test_carrier.py)
tests/_build/libcarrier_device.so: tests/device_shim/carrier_device.cu build/modes_signal.o build/modes_tables.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/carrier_device.cu -o tests/_build/carrier_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/carrier_device.o build/modes_signal.o build/modes_tables.o -cudart static
# the scan, frame-evaluation and weak-preamble kernels with a chosen SM count (tests/test_persistent_kernels.py)
SCAN_EVAL_OBJS := build/modes_scan2.o build/modes_eval_fused.o build/modes_kernels.o build/modes_weak.o build/modes_tables.o
tests/_build/libscan_eval_device.so: tests/device_shim/scan_eval_device.cu $(SCAN_EVAL_OBJS) $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/scan_eval_device.cu -o tests/_build/scan_eval_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/scan_eval_device.o $(SCAN_EVAL_OBJS) -cudart static
# the receiver pool's resampling and history launches on constructed jobs (tests/test_pool_input_rate.py)
tests/_build/libresample_pool_device.so: tests/device_shim/resample_pool_device.cu build/modes_resample.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/resample_pool_device.cu -o tests/_build/resample_pool_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/resample_pool_device.o build/modes_resample.o -cudart static
# the receiver pool's conversion launch on constructed jobs (tests/test_pool_input_format.py)
tests/_build/libconvert_pool_device.so: tests/device_shim/convert_pool_device.cu build/modes_resample.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/convert_pool_device.cu -o tests/_build/convert_pool_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/convert_pool_device.o build/modes_resample.o -cudart static
# the receiver pool's gather launch on constructed jobs (tests/test_pool_device_input.py)
tests/_build/libgather_pool_device.so: tests/device_shim/gather_pool_device.cu build/modes_resample.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/gather_pool_device.cu -o tests/_build/gather_pool_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/gather_pool_device.o build/modes_resample.o -cudart static
# the 16-bit input launches on chosen spans, and their timing (tests/test_input_format.py, scripts/input_format_time.py)
tests/_build/libinput_device.so: tests/device_shim/input_device.cu build/modes_resample.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/input_device.cu -o tests/_build/input_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/input_device.o build/modes_resample.o -cudart static
# the decimator, its frequency shift and the spectrum pass on chosen spans and pool jobs (tests/test_rate_kernels.py)
RATE_SPECTRUM_OBJS := build/modes_resample.o build/modes_spectrum.o
tests/_build/librate_spectrum_device.so: tests/device_shim/rate_spectrum_device.cu $(RATE_SPECTRUM_OBJS) $(CSRC)/modes_internal.h $(CSRC)/modes_resample_core.cuh $(CSRC)/modes_spectrum_core.cuh include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/rate_spectrum_device.cu -o tests/_build/rate_spectrum_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/rate_spectrum_device.o $(RATE_SPECTRUM_OBJS) -cudart static
# the device resolve with a chosen SM count, batch size and delivery capacity (tests/test_resolve_device.py)
tests/_build/libresolve_device.so: tests/device_shim/resolve_device.cu build/modes_resolve_gpu.o $(CSRC)/modes_internal.h include/modes_b200.h
	@mkdir -p tests/_build
	$(NVCC) $(NVFLAGS) -I$(CSRC) -c tests/device_shim/resolve_device.cu -o tests/_build/resolve_device.o
	$(NVCC) $(ARCH) -shared -o $@ tests/_build/resolve_device.o build/modes_resolve_gpu.o -cudart static

clean:
	rm -rf build tests/_build $(LIB) dump1090-b200

.PHONY: all oracle shim dshim clean
