# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/rsem-bam2wig and oracle/_ref/rsem-bam2readdepth, the UNMODIFIED
# reference tools, from $(REF)/bam2wig.cpp / $(REF)/bam2readdepth.cpp and $(REF)/wiggle.cpp with the reference
# Makefile's -O3 (its OBJS2 rule), linked with the htslib 1.3 that oracle/Makefile compiles into $(OUT)/libhts.a (run
# that first; build.py does).  Also installs the unmodified rsem-plot-transcript-wiggles and its module beside them, as
# the reference's `make install` does.  The tests compare bin/rsem-bam2wig and bin/rsem-bam2readdepth against these.
# Without $(REF) this is a no-op.
REF      ?= /root/reference
OUT      := _ref
CXX      := g++
FLAGS    := -std=gnu++98 -w -O3 -I$(REF) -I$(REF)/samtools-1.3/htslib-1.3

ifneq ($(wildcard $(REF)/wiggle.cpp),)
all: $(OUT)/rsem-bam2wig $(OUT)/rsem-bam2readdepth $(OUT)/rsem-plot-transcript-wiggles
else
all:
	@true
endif

$(OUT)/wiggle.o: $(REF)/wiggle.cpp $(OUT)/libhts.a
	$(CXX) $(FLAGS) -c $< -o $@

$(OUT)/rsem-bam2wig: $(REF)/bam2wig.cpp $(OUT)/wiggle.o $(OUT)/libhts.a
	$(CXX) $(FLAGS) $(REF)/bam2wig.cpp $(OUT)/wiggle.o $(OUT)/libhts.a -o $@ -pthread -static-libstdc++ -static-libgcc -lz

$(OUT)/rsem-bam2readdepth: $(REF)/bam2readdepth.cpp $(OUT)/wiggle.o $(OUT)/libhts.a
	$(CXX) $(FLAGS) $(REF)/bam2readdepth.cpp $(OUT)/wiggle.o $(OUT)/libhts.a -o $@ -pthread -static-libstdc++ -static-libgcc -lz

$(OUT)/rsem-plot-transcript-wiggles: $(REF)/rsem-plot-transcript-wiggles $(REF)/rsem_perl_utils.pm
	cp $(REF)/rsem-plot-transcript-wiggles $(REF)/rsem_perl_utils.pm $(OUT)/
	chmod u+w,a+x $(OUT)/rsem-plot-transcript-wiggles $(OUT)/rsem_perl_utils.pm

.PHONY: all
