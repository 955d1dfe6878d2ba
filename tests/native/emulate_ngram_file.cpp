// TEST INFRASTRUCTURE ONLY -- emulate_ngram.cpp (the CTA program with the library's own n-gram scorer, in the CPU
// emulation) over load_ngram_file, the loader ctcdec_scorer_create_arpa uses: ARPA text or a KenLM binary file.
// tests/test_kenlm_binary.py compiles this file into tests/native/_build/.  The product never builds or loads it.
#include "../../ctcdecode_b200/csrc/ngram_kenlm.h"
// emulate_ngram.cpp loads its model with load_arpa (ARPA text only); here that one call reads either form.  The
// loaders are declared above, so the name is only replaced in the harness's own code.
#define load_arpa load_ngram_file
#include "emulate_ngram.cpp"
#undef load_arpa
