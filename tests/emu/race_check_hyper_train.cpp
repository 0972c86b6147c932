// tests/emu/race_check_hyper_train.cpp — TEST INFRASTRUCTURE: data-race check of HypER's training-mode trunk kernels
// (kge_hyper_train.cuh: the bn0 output, the filters, z1 and dz passed between phases of a CTA through shared memory,
// global memory and __syncthreads; the CTA sums through a shared array; the float atomics of the scatters) under the
// host emulation, in a binary built with -fsanitize=thread.  The run itself is main() of emu_hyper_train.cpp (forward
// and backward over two groups whose queries share an entity and a relation).  The same source built with
// -DCUDA_EMU_NO_BARRIERS must be reported (positive control).
//
//   race_check_hyper_train          run the kernels
//   race_check_hyper_train probe    exit 64 without running them (is the sanitizer runtime usable?)
#define HYPER_TRAIN_RACE_MAIN
#include "emu_hyper_train.cpp"
