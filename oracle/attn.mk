# oracle/attn.mk — TEST INFRASTRUCTURE ONLY: the program behind the attention and KV-cache ops' tests, on top of oracle/decoders.mk (and
# through it oracle/Makefile's reference libraries):  make -C oracle -f attn.mk attn
#   _ref/libggml_attn_probe.so  FLASH_ATTN_EXT, SOFT_MAX and CPY-into-a-cache graphs on a named device (attn_probe.cpp), for ctypes
# Like everything in _ref/ it is git-ignored.
include decoders.mk

.PHONY: attn
attn: $(OUT)/libggml_attn_probe.so
