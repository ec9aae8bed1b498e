# oracle/llama.mk — TEST INFRASTRUCTURE ONLY: the programs behind the llama-family (rotary position embedding) tests, built on top of
# oracle/Makefile's reference libraries:  make -C oracle -f llama.mk llama
#   _ref/libggml_rope_probe.so  one-node ROPE graphs on a named device (rope_probe.cpp), for ctypes
#   _ref/llama-graph            a synthetic llama-architecture decoder on the reference's graph / scheduler API (llama_graph.cpp)
# Both are this repository's own code over the reference's public headers; like everything in _ref/ they are git-ignored.
include Makefile

.PHONY: llama
llama: $(OUT)/libggml_rope_probe.so $(OUT)/llama-graph

$(OUT)/libggml_rope_probe.so: rope_probe.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -shared -o $@ $< $(LINK)
$(OUT)/llama-graph: llama_graph.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -o $@ $< $(LINK)
