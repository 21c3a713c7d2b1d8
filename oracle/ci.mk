# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/rsem-calculate-credibility-intervals, the UNMODIFIED reference tool, from
# $(REF)/calcCI.cpp with the reference's flags for it (-O3 -ffast-math, reference Makefile:39,72-73).  The tests
# compare bin/rsem-calculate-credibility-intervals against it byte for byte.  Without $(REF) this is a no-op.
REF      ?= /root/reference
OUT      := _ref
CXX      := g++

ifneq ($(wildcard $(REF)/calcCI.cpp),)
all: $(OUT)/rsem-calculate-credibility-intervals
else
all:
	@true
endif

# compiled and linked in two steps like the reference build: -ffast-math on the compile only, so the link does not add
# crtfastmath.o (which would set flush-to-zero for the whole process)
$(OUT)/calcCI.o: $(REF)/calcCI.cpp
	mkdir -p $(OUT)
	$(CXX) -std=gnu++98 -w -O3 -ffast-math -I$(REF) -c $< -o $@

$(OUT)/rsem-calculate-credibility-intervals: $(OUT)/calcCI.o
	$(CXX) -pthread $< -o $@ -static-libstdc++ -static-libgcc

.PHONY: all
