# oracle/yolo.mk — TEST INFRASTRUCTURE ONLY: the programs behind the YOLO-style convolutional network's tests, on top of oracle/decoders.mk
# (and through it oracle/Makefile's reference libraries):  make -C oracle -f yolo.mk yolo
#   _ref/libggml_pool_probe.so  POOL_2D, UPSCALE, LEAKY_RELU and REPEAT graphs on a named device (pool_probe.cpp), for ctypes
#   _ref/yolo-graph             a synthetic YOLOv3-tiny (yolo_graph.cpp over decoder_harness.h)
#   _ref/yolov3-tiny            the reference's examples/yolo program, unmodified, on ggml-cpu
#   _ref/yolov3-tiny-b200       the same sources with -DGGML_USE_CUDA, so that ggml_backend_cuda_init binds this repository's plug-in
#   _ref/yolo/data/             the example's coco.names and label glyphs, which the program reads relative to its working directory
# Like everything in _ref/ they are git-ignored.
include decoders.mk

YOLO    := $(REF)/examples/yolo
YOLOSRC := $(YOLO)/yolov3-tiny.cpp $(YOLO)/yolo-image.cpp

.PHONY: yolo
yolo: $(OUT)/libggml_pool_probe.so $(OUT)/yolo-graph $(OUT)/yolov3-tiny $(OUT)/yolov3-tiny-b200 $(OUT)/yolo/data/STAMP

$(OUT)/yolov3-tiny: $(YOLOSRC) $(OUT)/libggml.so
	$(CXX) $(CXXFLAGS) -I$(REF)/examples -o $@ $(YOLOSRC) $(LINK)
$(OUT)/yolov3-tiny-b200: $(YOLOSRC) $(OUT)/libggml.so $(B200LIB)
	$(CXX) $(CXXFLAGS) -DGGML_USE_CUDA -I$(REF)/examples -o $@ $(YOLOSRC) $(LINK) $(B200LINK)
$(OUT)/yolo/data/STAMP: $(YOLO)/data/coco.names $(wildcard $(YOLO)/data/labels/*.png)
	@mkdir -p $(OUT)/yolo/data
	cp $(YOLO)/data/coco.names $(OUT)/yolo/data/
	cp -r $(YOLO)/data/labels $(OUT)/yolo/data/
	touch $@
