// TEST INFRASTRUCTURE ONLY -- emulate_readout.cpp (the read-out kernel's per-row function compiled for the CPU) over
// load_ngram_file, the loader ctcdec_scorer_create_arpa uses: ARPA text or a KenLM binary file.
// tests/test_kenlm_binary.py compiles this file into tests/native/_build/.  The product never builds or loads it.
#include "../../ctcdecode_b200/csrc/ngram_kenlm.h"
// emulate_readout.cpp loads its model with load_arpa (ARPA text only); here that one call reads either form.  The
// loaders are declared above, so the name is only replaced in the harness's own code.
#define load_arpa load_ngram_file
#include "emulate_readout.cpp"
#undef load_arpa
