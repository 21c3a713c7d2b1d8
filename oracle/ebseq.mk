# TEST INFRASTRUCTURE ONLY.  Builds
#   (1) oracle/_ref/rsem-for-ebseq-calculate-clustering-info, the UNMODIFIED reference tool, from
#       $(REF)/EBSeq/calcClusteringInfo.cpp with the flags of the reference's EBSeq/Makefile (g++ -O3 -Wall); the tests
#       compare bin/rsem-for-ebseq-calculate-clustering-info against it byte for byte.  Without $(REF) this part is a
#       no-op;
#   (2) oracle/libkmer_oracle.so, our plain-C restatement of the tool's counts (oracle/kmer_oracle.c).
REF      ?= /root/reference
OUT      := _ref
CXX      := g++
CC       := gcc

ifneq ($(wildcard $(REF)/EBSeq/calcClusteringInfo.cpp),)
all: libkmer_oracle.so $(OUT)/rsem-for-ebseq-calculate-clustering-info
else
all: libkmer_oracle.so
endif

libkmer_oracle.so: kmer_oracle.c
	$(CC) -O2 -fPIC -shared -std=c11 -Wall -o $@ $<

# static libstdc++/libgcc so the binary runs unchanged on other machines with the same CPU architecture
$(OUT)/rsem-for-ebseq-calculate-clustering-info: $(REF)/EBSeq/calcClusteringInfo.cpp
	mkdir -p $(OUT)
	$(CXX) -O3 -Wall $< -o $@ -static-libstdc++ -static-libgcc

.PHONY: all
