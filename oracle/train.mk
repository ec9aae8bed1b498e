# oracle/train.mk — TEST INFRASTRUCTURE ONLY: the programs behind the training ops' tests, on top of oracle/decoders.mk (and through it
# oracle/Makefile's reference libraries):  make -C oracle -f train.mk train
#   _ref/libggml_train_probe.so  OUT_PROD, CROSS_ENTROPY_LOSS, CROSS_ENTROPY_LOSS_BACK, OPT_STEP_ADAMW, ARGMAX, COUNT_EQUAL, SUM,
#                                REPEAT_BACK and STEP graphs on a named device (train_probe.cpp), for ctypes
#   _ref/train-graph             a synthetic 784-500-10 classifier trained through ggml-opt.h on ggml_backend_sched (train_graph.cpp)
# Like everything in _ref/ they are git-ignored.
include decoders.mk

.PHONY: train
train: $(OUT)/libggml_train_probe.so $(OUT)/train-graph

$(OUT)/train-graph: train_graph.cpp $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -o $@ $< $(LINK)
