# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/rsem-tbam2gbam, the UNMODIFIED reference tool, from $(REF)/tbam2gbam.cpp
# and $(REF)/SamHeader.cpp with the reference Makefile's -O2, linked with the htslib 1.3 that oracle/Makefile compiles
# into $(OUT)/libhts.a (run that first; build.py does).  The tests compare bin/rsem-tbam2gbam against it.  Without $(REF)
# this is a no-op.
REF      ?= /root/reference
OUT      := _ref
CXX      := g++

ifneq ($(wildcard $(REF)/tbam2gbam.cpp),)
all: $(OUT)/rsem-tbam2gbam
else
all:
	@true
endif

$(OUT)/rsem-tbam2gbam: $(REF)/tbam2gbam.cpp $(REF)/SamHeader.cpp $(OUT)/libhts.a
	$(CXX) -std=gnu++98 -w -pthread -O2 -I$(REF) -I$(REF)/samtools-1.3/htslib-1.3 $(REF)/tbam2gbam.cpp $(REF)/SamHeader.cpp \
	    $(OUT)/libhts.a -o $@ -pthread -static-libstdc++ -static-libgcc -lz

.PHONY: all
