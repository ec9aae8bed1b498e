# oracle/rwkv.mk — TEST INFRASTRUCTURE ONLY: the programs behind the RWKV-6 tests, built on top of oracle/Makefile's reference libraries:
#   make -C oracle -f rwkv.mk rwkv
#   _ref/libggml_wkv_probe.so  one-node RWKV_WKV6 / GATED_LINEAR_ATTN / SQR / SQRT graphs on a named device (wkv_probe.cpp), for ctypes
#   _ref/rwkv-graph            a synthetic RWKV-6 decoder on the reference's graph / scheduler API (rwkv_graph.cpp)
# Both are this repository's own code over the reference's public headers; like everything in _ref/ they are git-ignored.
include Makefile

.PHONY: rwkv
rwkv: $(OUT)/libggml_wkv_probe.so $(OUT)/rwkv-graph

$(OUT)/libggml_wkv_probe.so: wkv_probe.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -shared -o $@ $< $(LINK)
$(OUT)/rwkv-graph: rwkv_graph.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -o $@ $< $(LINK)
