// tests/emu/race_check_tucker.cpp — TEST INFRASTRUCTURE: data-race check of TuckER's trunk kernels (kge_tucker.cuh:
// the row and the two reductions of the forward in shared memory; the backward's shared rows reused across phases
// and its float atomics) under the host emulation, in a binary built with -fsanitize=thread.  The run itself is
// main() of emu_tucker.cpp (cores, forward, backward, cores' backward on a batch whose queries share a relation
// and an entity).  The same source built with -DCUDA_EMU_NO_BARRIERS must be reported (positive control).
//
//   race_check_tucker          run the kernels
//   race_check_tucker probe    exit 64 without running them (is the sanitizer runtime usable?)
#define TUCKER_RACE_MAIN
#include "emu_tucker.cpp"
