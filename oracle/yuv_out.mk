# TEST INFRASTRUCTURE - builds _ref/libyuv_out_ref.so: the reference's vendored libyuv (core/3rdparty/libyuv, version 1744), portable C
# rows only, compiled from the sources where they lie (nothing is copied), plus yuv_out_shim.cpp (RGBA8 -> NV12 / NV21 / I420). The
# tests compare the numpy restatement of that conversion (yuv_out.py) with it when it exists; without the reference tree (or when it
# does not compile) nothing is built, and they use tests/golden/yuv_out_golden.npz alone.
# The reference checkout: $(SNNB_REFERENCE) when set, else the same default as Makefile.
REF ?= $(if $(SNNB_REFERENCE),$(SNNB_REFERENCE),/root/reference)
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
YUV := $(REF)/core/3rdparty/libyuv
YUV_SRC := $(addprefix $(YUV)/source/,convert.cc convert_from_argb.cc row_common.cc row_any.cc cpu_id.cc planar_functions.cc \
  scale_common.cc scale.cc scale_any.cc)

yuv_out:
	@if [ -d $(YUV)/source ]; then \
	  mkdir -p _ref && \
	  $(CXX) -std=c++17 -O2 -fPIC -shared -w -DLIBYUV_DISABLE_X86 -DLIBYUV_DISABLE_NEON -Wl,--no-undefined -I$(YUV)/include \
	    yuv_out_shim.cpp $(YUV_SRC) -o _ref/libyuv_out_ref.so && echo "built _ref/libyuv_out_ref.so" \
	    || echo "libyuv_out_ref.so not built: the tests compare with tests/golden/yuv_out_golden.npz only"; \
	else echo "reference libyuv absent: keeping prebuilt _ref (if any)"; fi

.PHONY: yuv_out
