# Same commands as __graft_entry__.build(): the sm_90a shared library (all kernels + C ABI) and the GEMM self-test.
NVCC      ?= nvcc
NVCCFLAGS ?= -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17
SRCS      := csrc/otb_host.cu csrc/otb_gemm.cu csrc/otb_attn.cu csrc/otb_norm.cu csrc/otb_fp32.cu csrc/otb_loss.cu csrc/otb_attn_lm.cu csrc/otb_data.cu csrc/otb_persimmon.cu csrc/otb_xattn_fused.cu csrc/otb_llama.cu csrc/otb_fp32_bwd.cu csrc/otb_lora.cu csrc/otb_decode.cu
LIB       := otter_b200/lib/libotter_b200.so

all: $(LIB) build/selftest_gemm

$(LIB): $(SRCS) csrc/otb_common.cuh csrc/otb_host.h include/otter_b200.h
	@mkdir -p $(dir $@)
	$(NVCC) $(NVCCFLAGS) -Xcompiler -fPIC --threads 4 -shared -o $@ $(SRCS)

build/selftest_gemm: csrc/selftest_gemm.cu $(LIB)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -o $@ $< -Lotter_b200/lib -lotter_b200 -Xlinker -rpath -Xlinker '$$ORIGIN/../otter_b200/lib'

sass-check: $(LIB)
	cuobjdump -sass $(LIB) | grep -oE "HGMMA[.A-Z0-9]*|UTMALDG[.A-Z0-9]*|UTMASTG[.A-Z0-9]*" | sort | uniq -c

clean:
	rm -f $(LIB) build/selftest_gemm

.PHONY: all sass-check clean
