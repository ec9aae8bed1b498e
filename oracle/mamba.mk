# oracle/mamba.mk — TEST INFRASTRUCTURE ONLY: the programs behind the Mamba (selective state-space) tests, built on top of oracle/Makefile's
# reference libraries:  make -C oracle -f mamba.mk mamba
#   _ref/libggml_ssm_probe.so  one-node CONCAT / SSM_CONV / SSM_SCAN graphs on a named device (ssm_probe.cpp), for ctypes
#   _ref/mamba-graph           a synthetic Mamba decoder on the reference's graph / scheduler API (mamba_graph.cpp)
# Both are this repository's own code over the reference's public headers; like everything in _ref/ they are git-ignored.
include Makefile

.PHONY: mamba
mamba: $(OUT)/libggml_ssm_probe.so $(OUT)/mamba-graph

$(OUT)/libggml_ssm_probe.so: ssm_probe.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -shared -o $@ $< $(LINK)
$(OUT)/mamba-graph: mamba_graph.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -o $@ $< $(LINK)
