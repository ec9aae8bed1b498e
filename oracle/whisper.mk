# oracle/whisper.mk — TEST INFRASTRUCTURE ONLY: the programs behind the convolutional front end's tests, on top of oracle/decoders.mk
# (and through it oracle/Makefile's reference libraries):  make -C oracle -f whisper.mk whisper
#   _ref/libggml_conv_probe.so  IM2COL, f16 x f16 MUL_MAT and ggml_conv_1d graphs on a named device (conv_probe.cpp), for ctypes
#   _ref/whisper-graph          a synthetic Whisper-style encoder-decoder (whisper_graph.cpp over decoder_harness.h)
# Like everything in _ref/ they are git-ignored.
include decoders.mk

.PHONY: whisper
whisper: $(OUT)/libggml_conv_probe.so $(OUT)/whisper-graph
