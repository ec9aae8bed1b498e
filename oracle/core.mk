# oracle/core.mk — TEST INFRASTRUCTURE ONLY: the program behind the small ops' tests, on top of oracle/decoders.mk (and through it
# oracle/Makefile's reference libraries):  make -C oracle -f core.mk core
#   _ref/libggml_core_probe.so  GET_ROWS, the broadcast binary ops, the norms, SCALE / DIAG_MASK_INF, the unary ops, the float CPY and the
#                               two fused chains as graphs on a named device (core_probe.cpp), for ctypes
# Like everything in _ref/ it is git-ignored.
include decoders.mk

.PHONY: core
core: $(OUT)/libggml_core_probe.so
