# TEST INFRASTRUCTURE (oracle), stage 0.  `make -C oracle -f stage0.mk` builds, from the
# reference sources where they lie under $(REF) (read-only, nothing is copied), into oracle/_ref/:
#   fastq-extractor      stock stage-0 binary (FastqExtractor.cpp)
#   fastq-extractor-gpu  the drop-in of integration/Makefile: FastqExtractor.cpp as
#                        integration/make_extractor_main.py patches it, with
#                        integration/t4_extractor_adapter.hpp force-included, linked against
#                        ../trust4_b200/libtrust4_b200.so (which must exist first)
# so that tests/test_gpu_extractor.py and bench/stage0_extract.py run where the reference
# sources are absent.  One g++ command per target with the reference's flags (-O3 -g,
# -lpthread -lz); the patched driver source goes to a temporary directory and is removed.
REF ?= /root/reference
OUT = _ref
CXX = g++
CXXFLAGS = -O3 -g -w

all: $(OUT)/fastq-extractor $(OUT)/fastq-extractor-gpu

$(OUT):
	mkdir -p $(OUT)

$(OUT)/fastq-extractor: | $(OUT)
	$(CXX) $(CXXFLAGS) -o $@ $(REF)/FastqExtractor.cpp -lpthread -lz

# rpath $ORIGIN/../../trust4_b200 resolves from oracle/_ref/ as from integration/_build/
$(OUT)/fastq-extractor-gpu: ../trust4_b200/libtrust4_b200.so ../integration/t4_extractor_adapter.hpp ../include/trust4_b200.h \
		../integration/make_extractor_main.py | $(OUT)
	tmp=$$(mktemp -d) && python3 ../integration/make_extractor_main.py $(REF)/FastqExtractor.cpp $$tmp/extractor_main.cpp && \
	$(CXX) $(CXXFLAGS) -I$(REF) -I../include -include ../integration/t4_extractor_adapter.hpp -o $@ $$tmp/extractor_main.cpp \
		-L../trust4_b200 -ltrust4_b200 -Wl,-rpath,'$$ORIGIN/../../trust4_b200' -lpthread -lz; st=$$?; rm -rf $$tmp; exit $$st

.PHONY: all
