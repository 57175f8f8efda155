# Build libnvcomp.so (H100 / sm_90a only) and the CPU oracle.
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -Iinclude -Invcomp_b200/csrc
SRC_DIR   := nvcomp_b200/csrc
BUILD_DIR := build
LIB       := nvcomp_b200/lib/libnvcomp.so
SRCS      := $(wildcard $(SRC_DIR)/*.cu)
OBJS      := $(patsubst $(SRC_DIR)/%.cu,$(BUILD_DIR)/%.o,$(SRCS))
HDRS      := $(wildcard $(SRC_DIR)/*.cuh) $(wildcard $(SRC_DIR)/*.h) $(wildcard include/nvcomp/*.h) $(wildcard include/nvcomp/*.hpp) $(wildcard include/*.hpp) \
            $(wildcard include/nvcomp/device/*.cuh) $(wildcard include/nvcomp/device/detail/*.cuh)

ORACLE_SRCS := $(wildcard oracle/*.c)
ORACLE_LIB  := oracle/liboracle.so

TESTS_BIN := build/tests/hlif_test build/tests/deflate_hlif_test
# kernels over the warp-level ANS device API (include/nvcomp/device/ans.cuh), loaded by the tests with ctypes
ANS_DEVICE_LIB := build/tests/libans_device.so
# kernels over the warp-level Bitcomp device API (include/nvcomp/device/bitcomp.cuh), loaded the same way
BITCOMP_DEVICE_LIB := build/tests/libbitcomp_device.so
# kernels over the warp-level Cascaded device API (include/nvcomp/device/cascaded.cuh), loaded the same way
CASCADED_DEVICE_LIB := build/tests/libcascaded_device.so
# kernels over the warp-level LZ4 and Snappy device APIs (include/nvcomp/device/{lz4,snappy}.cuh), loaded the same way
LZ_DEVICE_LIB := build/tests/liblz_device.so
# kernels over the warp-level Deflate, Gzip and Zstd device APIs (include/nvcomp/device/{deflate,gzip,zstd}.cuh), loaded
# the same way
DZ_DEVICE_LIB := build/tests/libdeflate_zstd_device.so
# kernels over zstd::compress_warp (include/nvcomp/device/zstd.cuh), loaded the same way
ZC_DEVICE_LIB := build/tests/libzstd_compress_device.so
# kernels over the warp-level LZ4 frame device API (include/nvcomp/device/lz4frame.cuh), loaded the same way
LZ4F_DEVICE_LIB := build/tests/liblz4frame_device.so build/tests/liblz4frame_device_rdc.so
# one library linked from two translation units that include all eight device headers, plain and with -rdc=true: the
# headers must not define functions with external, non-inline linkage (tests/cpp/device_headers_link.cu)
LINK_LIBS := build/tests/libdevice_headers_link.so build/tests/libdevice_headers_link_rdc.so
# extern "C" dispatch onto the C++ managers (nvcomp::*Manager, create_manager), loaded the same way
HLIF_SHIM_LIB := build/tests/libhlif_shim.so

# host warp emulator (test infrastructure): the warp-level decode headers compiled with g++, PTX shadowed
EMU_LIB  := tests/emu/libemu_lz.so
EMU_SRCS := tests/emu/emu_cuda.cpp tests/emu/emu_lz.cpp tests/emu/emu_inflate.cpp tests/emu/emu_deflate.cpp \
            tests/emu/emu_zstd.cpp tests/emu/emu_zstd_encode.cpp tests/emu/emu_lz_encode.cpp \
            tests/emu/emu_lz4frame.cpp

all: $(LIB) $(ORACLE_LIB) $(TESTS_BIN) $(ANS_DEVICE_LIB) $(BITCOMP_DEVICE_LIB) $(CASCADED_DEVICE_LIB) $(LZ_DEVICE_LIB) $(DZ_DEVICE_LIB) $(ZC_DEVICE_LIB) $(LZ4F_DEVICE_LIB) $(LINK_LIBS) $(HLIF_SHIM_LIB) $(EMU_LIB)

$(EMU_LIB): $(EMU_SRCS) $(wildcard tests/emu/*.h) $(wildcard tests/emu/*.cuh) $(wildcard tests/emu/nvcomp/device/detail/*.cuh) $(HDRS)
	g++ -std=c++17 -O2 -g -fPIC -shared -Wall -Wno-unknown-pragmas -Wno-unused-function \
	    -Itests/emu -I$(SRC_DIR) -Iinclude -I/usr/local/cuda/include $(EMU_SRCS) -o $@

$(BUILD_DIR)/%.o: $(SRC_DIR)/%.cu $(HDRS)
	@mkdir -p $(BUILD_DIR)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(BUILD_DIR)/$*.ptxas.log || (cat $(BUILD_DIR)/$*.ptxas.log; exit 1)

$(LIB): $(OBJS)
	@mkdir -p nvcomp_b200/lib
	$(NVCC) $(ARCH) -shared -Xlinker -soname=libnvcomp.so -o $@ $(OBJS) -cudart static

$(ORACLE_LIB): $(ORACLE_SRCS) $(wildcard oracle/*.h)
	gcc -O3 -march=x86-64-v2 -fPIC -shared -Wall -o $@ $(ORACLE_SRCS) -ldl -lpthread

build/tests/%: tests/cpp/%.cu $(LIB) $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -std=c++17 -O2 -Iinclude $< -o $@ -Lnvcomp_b200/lib -lnvcomp -Xlinker '-rpath=$$ORIGIN/../../nvcomp_b200/lib'

$(ANS_DEVICE_LIB): tests/cpp/ans_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/libans_device.ptxas.log || (cat build/tests/libans_device.ptxas.log; exit 1)

$(BITCOMP_DEVICE_LIB): tests/cpp/bitcomp_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/libbitcomp_device.ptxas.log || (cat build/tests/libbitcomp_device.ptxas.log; exit 1)

$(CASCADED_DEVICE_LIB): tests/cpp/cascaded_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/libcascaded_device.ptxas.log || (cat build/tests/libcascaded_device.ptxas.log; exit 1)

$(LZ_DEVICE_LIB): tests/cpp/lz_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/liblz_device.ptxas.log || (cat build/tests/liblz_device.ptxas.log; exit 1)

$(DZ_DEVICE_LIB): tests/cpp/deflate_zstd_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/libdeflate_zstd_device.ptxas.log || (cat build/tests/libdeflate_zstd_device.ptxas.log; exit 1)

$(ZC_DEVICE_LIB): tests/cpp/zstd_compress_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/libzstd_compress_device.ptxas.log || (cat build/tests/libzstd_compress_device.ptxas.log; exit 1)

build/tests/liblz4frame_device.so: tests/cpp/lz4frame_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared -Xptxas -v $< -o $@ \
	    2> build/tests/liblz4frame_device.ptxas.log || (cat build/tests/liblz4frame_device.ptxas.log; exit 1)

# the same kernels built with -rdc=true and linked with a second translation unit over the same headers
build/tests/lz4frame_rdc_%.o: tests/cpp/lz4frame_device_kernels.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -rdc=true $(if $(filter 2,$*),-DLZ4F_LINK_ONLY) -c $< -o $@

build/tests/liblz4frame_device_rdc.so: build/tests/lz4frame_rdc_1.o build/tests/lz4frame_rdc_2.o
	$(NVCC) $(ARCH) -rdc=true -shared $^ -o $@

build/tests/link_tu%.o: tests/cpp/device_headers_link.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -DLINK_TU=$* -c $< -o $@

build/tests/link_rdc_tu%.o: tests/cpp/device_headers_link.cu $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O3 -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -rdc=true -DLINK_TU=$* -c $< -o $@

build/tests/libdevice_headers_link.so: build/tests/link_tu1.o build/tests/link_tu2.o
	$(NVCC) $(ARCH) -shared $^ -o $@

build/tests/libdevice_headers_link_rdc.so: build/tests/link_rdc_tu1.o build/tests/link_rdc_tu2.o
	$(NVCC) $(ARCH) -rdc=true -shared $^ -o $@

$(HLIF_SHIM_LIB): tests/cpp/hlif_shim.cu $(LIB) $(HDRS)
	@mkdir -p build/tests
	$(NVCC) $(ARCH) -O2 -std=c++17 -Xcompiler -fPIC,-Wall -Iinclude -shared $< -o $@ \
	    -Lnvcomp_b200/lib -lnvcomp -Xlinker '-rpath=$$ORIGIN/../../nvcomp_b200/lib'

clean:
	rm -rf $(BUILD_DIR) $(LIB) $(ORACLE_LIB)

.PHONY: all clean
