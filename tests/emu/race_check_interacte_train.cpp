// tests/emu/race_check_interacte_train.cpp — TEST INFRASTRUCTURE: data-race check of InteractE's training-mode trunk
// kernels (kge_interacte_train.cuh: the padded bn0 outputs, the filter bank, z1, dz1, d img and the inverse
// permutations passed between phases of a CTA through shared memory, global memory and __syncthreads; the CTA sums
// through a shared array; the float atomics of the scatter) under the host emulation, in a binary built with
// -fsanitize=thread.  The run itself is main() of emu_interacte_train.cpp (forward and backward over two groups whose
// queries share an entity and a relation).  The same source built with -DCUDA_EMU_NO_BARRIERS must be reported
// (positive control).
//
//   race_check_interacte_train          run the kernels
//   race_check_interacte_train probe    exit 64 without running them (is the sanitizer runtime usable?)
#define INTERACTE_TRAIN_RACE_MAIN
#include "emu_interacte_train.cpp"
