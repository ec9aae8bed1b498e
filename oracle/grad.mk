# oracle/grad.mk — TEST INFRASTRUCTURE ONLY: the program behind MUL_MAT's gradient tests:  make -C oracle -f grad.mk grad
#   _ref/libggml_grad_probe.so  MUL_MAT's backward graph on a named device, with test-backend-ops' numerical gradient (grad_probe.cpp),
#                               for ctypes
# It needs only the reference's public headers and the libraries oracle/Makefile built into _ref/, so it also builds where the reference
# tree is absent but _ref/ is present: the headers then come from the copy oracle/Makefile staged in _ref/ggml-src.  Like everything in
# _ref/ it is git-ignored.
REF      ?= /root/reference
OUT      := _ref
CXX      := g++
HDRS     := $(if $(wildcard $(REF)/include/ggml.h),$(REF)/include,$(OUT)/ggml-src/include)
CXXFLAGS := -std=c++17 -O3 -DNDEBUG -fPIC -pthread -DGGML_SHARED -I$(HDRS)
LINK     := -L$(OUT) -lggml -lggml-cpu -lggml-base -Wl,-rpath,'$$ORIGIN' -lm -pthread

.PHONY: grad
grad: $(OUT)/libggml_grad_probe.so

$(OUT)/libggml_grad_probe.so: grad_probe.cpp probe_harness.h $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -shared -o $@ $< $(LINK)
