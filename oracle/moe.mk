# oracle/moe.mk — TEST INFRASTRUCTURE ONLY: the programs behind the mixture-of-experts tests, built on top of oracle/Makefile's reference
# libraries:  make -C oracle -f moe.mk moe
#   _ref/libggml_moe_probe.so  one-node ARGSORT / SUM_ROWS graphs on a named device (moe_probe.cpp), for ctypes
#   _ref/moe-graph             a synthetic mixture-of-experts decoder on the reference's graph / scheduler API (moe_graph.cpp)
# Both are this repository's own code over the reference's public headers; like everything in _ref/ they are git-ignored.
include Makefile

.PHONY: moe
moe: $(OUT)/libggml_moe_probe.so $(OUT)/moe-graph

$(OUT)/libggml_moe_probe.so: moe_probe.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -shared -o $@ $< $(LINK)
$(OUT)/moe-graph: moe_graph.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -o $@ $< $(LINK)
