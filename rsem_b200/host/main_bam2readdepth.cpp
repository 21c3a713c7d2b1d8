// bin/rsem-bam2readdepth: drop-in for the reference's tool of that name (bam2readdepth.cpp, wiggle.cpp), which
// rsem-plot-transcript-wiggles runs on the sorted transcript BAM.
//
//   rsem-bam2readdepth sorted_bam_input readdepth_output
//
// Stdout, the exit status and the read-depth file are the reference's.  The per-base sums run on the device (K11), the
// formatting on host threads (host/wiggle.cpp).  Differences: inputs the reference has no defined result for (a mapped
// record outside the header's targets or at a negative position, an M operation past its target's end, an optional
// field of unknown type or cut short before the first ZW) stop the run with a message and exit status 255.  CRAM input
// is refused.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>

#include "host.hpp"

using namespace host;

int main(int argc, char* argv[]) {
    if (argc != 3) {
        printf("Usage: rsem-bam2readdepth sorted_bam_input readdepth_output\n");
        exit(-1);
    }
    if (const char* e = getenv("RSEM_B200_IO_THREADS")) g_io_threads = atoi(e);
    else g_io_threads = (int)std::thread::hardware_concurrency();
    g_io_threads = std::max(1, g_io_threads);

    FILE* fo = fopen(argv[2], "w");
    if (!fo) die(std::string("Cannot write to ") + argv[2] + "!");
    setvbuf(fo, nullptr, _IOFBF, 1 << 22);
    run_wiggles("rsem-bam2readdepth", argv[1], false, false, fo);
    if (fclose(fo) != 0) die(std::string("rsem-bam2readdepth: cannot write ") + argv[2]);
    return 0;
}
