# Plain-make entry points for integrators who do not want to go through Python (python -m hotstuff_b200.build does the same).
NVCC ?= nvcc
NVCCFLAGS ?= -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared -diag-suppress 550
CSRC := hotstuff_b200/csrc

.PHONY: all lib oracle hostemu test-cpu clean
all: lib oracle hostemu

lib: hotstuff_b200/libhs_crypto.so
hotstuff_b200/libhs_crypto.so: $(CSRC)/hs_engine.cu $(CSRC)/hs_ingest.cpp $(CSRC)/hs_multi.cpp $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/hs_crypto.h
	$(NVCC) $(NVCCFLAGS) -o $@ $(CSRC)/hs_engine.cu $(CSRC)/hs_ingest.cpp $(CSRC)/hs_multi.cpp

# test infrastructure only (never linked into the product)
oracle:
	$(MAKE) -C oracle
hostemu: tests/hostemu/libhs_hostemu.so
tests/hostemu/libhs_hostemu.so: tests/hostemu/hostemu.cpp $(wildcard $(CSRC)/*.cuh)
	g++ -O2 -std=c++17 -fPIC -shared -DHS_HOST_EMU -Wno-unknown-pragmas -o $@ $<

test-cpu: all
	python -m pytest tests -x -q -m "not gpu"

clean:
	rm -f hotstuff_b200/libhs_crypto.so oracle/libhs_oracle.so tests/hostemu/libhs_hostemu.so tests/cpp/crypto_tests
