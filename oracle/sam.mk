# oracle/sam.mk — TEST INFRASTRUCTURE ONLY: the programs behind the Segment-Anything-style tests, on top of oracle/decoders.mk (and through it
# oracle/Makefile's reference libraries):  make -C oracle -f sam.mk sam
#   _ref/libggml_sam_probe.so  WIN_PART, WIN_UNPART, GET_REL_POS, ADD_REL_POS, CONV_TRANSPOSE_2D, SIN and COS graphs on a named device
#                              (sam_probe.cpp), for ctypes
#   _ref/sam-graph             a synthetic SAM image encoder (ViT-B and a small one) and prompt encoder + mask decoder (sam_graph.cpp over
#                              decoder_harness.h)
# Like everything in _ref/ they are git-ignored.
include decoders.mk

.PHONY: sam
sam: $(OUT)/libggml_sam_probe.so $(OUT)/sam-graph
