// tests/emu/race_check_acre_train.cpp — TEST INFRASTRUCTURE: data-race check of AcrE's training-mode trunk kernels
// (kge_acre_train.cuh: v, the conv maps, the weight banks, the serial backward's two map slots that swap roles across
// its three layers, dimg and the CTA sums passed between phases of a CTA through shared memory, global memory and
// __syncthreads; the float atomics of the scatter) under the host emulation, in a binary built with -fsanitize=thread.
// The run itself is main() of emu_acre_train.cpp (forward and backward of both ways over two groups whose queries
// share an entity and a relation).  The same source built with -DCUDA_EMU_NO_BARRIERS must be reported (positive
// control).
//
//   race_check_acre_train          run the kernels
//   race_check_acre_train probe    exit 64 without running them (is the sanitizer runtime usable?)
#define ACRE_TRAIN_RACE_MAIN
#include "emu_acre_train.cpp"
