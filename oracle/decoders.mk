# oracle/decoders.mk — TEST INFRASTRUCTURE ONLY: the programs behind the decoder-graph tests, built on top of oracle/Makefile's reference
# libraries:  make -C oracle -f decoders.mk decoders  (or one family: llama | moe | mamba | rwkv)
#   _ref/libggml_X_probe.so  one-node graphs on a named device (X_probe.cpp), for ctypes: ROPE (rope); ARGSORT / SUM_ROWS (moe);
#                            CONCAT / SSM_CONV / SSM_SCAN (ssm); RWKV_WKV6 / GATED_LINEAR_ATTN / SQR / SQRT (wkv)
#                            The rule below builds every family's probe over probe_harness.h, those of the .mk files that
#                            include this one too
#   _ref/X-graph             a synthetic decoder on the reference's graph / scheduler API (X_graph.cpp over decoder_harness.h):
#                            llama-architecture (llama), mixture-of-experts (moe), Mamba (mamba), RWKV-6 (rwkv)
# All are this repository's own code over the reference's public headers; like everything in _ref/ they are git-ignored.
include Makefile

.PHONY: decoders llama moe mamba rwkv
decoders: llama moe mamba rwkv
llama: $(OUT)/libggml_rope_probe.so $(OUT)/llama-graph
moe: $(OUT)/libggml_moe_probe.so $(OUT)/moe-graph
mamba: $(OUT)/libggml_ssm_probe.so $(OUT)/mamba-graph
rwkv: $(OUT)/libggml_wkv_probe.so $(OUT)/rwkv-graph

$(OUT)/libggml_%_probe.so: %_probe.cpp probe_harness.h $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -shared -o $@ $< $(LINK)
$(OUT)/%-graph: %_graph.cpp decoder_harness.h $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -o $@ $< $(LINK)
