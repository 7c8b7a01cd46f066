# TEST INFRASTRUCTURE — encodec.cpp's three example programs, compiled UNCHANGED from the reference tree against this project's
# include/ and linked with -lbark_b200 instead of encodec + ggml: the proof that encodec.cpp callers switch by changing only the
# include path and the library.
#
#   make -C oracle -f encodec_examples.mk [REF=<bark.cpp source tree>] [OUT=<dir>]
#                 -> $(OUT)/encodec_compress, encodec_decompress, encodec_main   (default OUT: oracle/_ref, git-ignored)
REF      ?= $(or $(BARK_REFERENCE_DIR),/root/reference)
EX       := $(REF)/encodec.cpp/examples
OUT      ?= _ref
LIBDIR   := $(abspath ../bark.cpp_b200)
CXXFLAGS := -O2 -std=c++17 -w -I$(abspath ../include) -I$(EX)
LDFLAGS  := -L$(LIBDIR) -lbark_b200 -Wl,-rpath,'$$ORIGIN/../../bark.cpp_b200' -pthread   # found from oracle/_ref wherever the tree lies

.PHONY: examples
examples: $(OUT)/encodec_compress $(OUT)/encodec_decompress $(OUT)/encodec_main

$(OUT):
	mkdir -p $(OUT)
$(OUT)/encodec_common.o: $(EX)/common.cpp | $(OUT)
	g++ $(CXXFLAGS) -c $< -o $@
$(OUT)/encodec_%: $(EX)/%/main.cpp $(OUT)/encodec_common.o $(LIBDIR)/libbark_b200.so ../include/encodec.h | $(OUT)
	g++ $(CXXFLAGS) $< $(OUT)/encodec_common.o -o $@ $(LDFLAGS)
