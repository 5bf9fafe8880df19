# TEST INFRASTRUCTURE - builds _ref/libyuv10_ref.so: the reference's vendored libyuv (core/3rdparty/libyuv, version 1744), portable C
# rows only, compiled from the sources where they lie (nothing is copied), plus yuv10_shim.cpp. The tests compare the numpy restatement
# of the 10-bit rows and the BT.2020 / full-range BT.601 matrices (yuv10.py) with it when it exists; without the reference tree (or when
# it does not compile) nothing is built, and they use tests/golden/yuv10_golden.npz alone.
# The reference checkout: $(SNNB_REFERENCE) when set, else the same default as Makefile.
REF ?= $(if $(SNNB_REFERENCE),$(SNNB_REFERENCE),/root/reference)
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
YUV := $(REF)/core/3rdparty/libyuv
YUV_SRC := $(addprefix $(YUV)/source/,row_common.cc cpu_id.cc)

yuv10:
	@if [ -d $(YUV)/source ]; then \
	  mkdir -p _ref && \
	  $(CXX) -std=c++17 -O2 -fPIC -shared -w -DLIBYUV_DISABLE_X86 -DLIBYUV_DISABLE_NEON -Wl,--no-undefined -I$(YUV)/include \
	    yuv10_shim.cpp $(YUV_SRC) -o _ref/libyuv10_ref.so && echo "built _ref/libyuv10_ref.so" \
	    || echo "libyuv10_ref.so not built: the tests compare with tests/golden/yuv10_golden.npz only"; \
	else echo "reference libyuv absent: keeping prebuilt _ref (if any)"; fi

.PHONY: yuv10
