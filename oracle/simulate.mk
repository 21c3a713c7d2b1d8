# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/rsem-simulate-reads, the UNMODIFIED reference simulator, from
# $(REF)/simulation.cpp with the reference's flags for it (-O3 -ffast-math, reference Makefile:39,72-73).  The tests
# compare bin/rsem-simulate-reads against it byte for byte.  Without $(REF) this is a no-op.
REF      ?= /root/reference
OUT      := _ref
CXX      := g++

ifneq ($(wildcard $(REF)/simulation.cpp),)
all: $(OUT)/rsem-simulate-reads
else
all:
	@true
endif

# compiled and linked in two steps like the reference build: -ffast-math on the compile only, so the link does not add
# crtfastmath.o (which would set flush-to-zero for the whole process)
$(OUT)/simulation.o: $(REF)/simulation.cpp
	mkdir -p $(OUT)
	$(CXX) -std=gnu++98 -w -O3 -ffast-math -I$(REF) -c $< -o $@

$(OUT)/rsem-simulate-reads: $(OUT)/simulation.o
	$(CXX) $< -o $@ -static-libstdc++ -static-libgcc

.PHONY: all
