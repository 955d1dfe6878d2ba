# TEST INFRASTRUCTURE ONLY.  Builds
#   _ref/build_binary       -- KenLM's own lm/build_binary_main.cc, compiled where it lies under $(REF) and linked with
#                              the KenLM objects of ./Makefile (included below, so the objects are shared).
# tests/test_kenlm_binary.py and tests/test_gpu_kenlm_binary.py run it to write binary models (probing, trie, quantized
# and array-compressed tries) of the committed ARPA fixtures into a temporary directory, always with -S 64M -T <tmp> so
# that building a trie sorts in a small local buffer; no binary model is committed, and the tests skip without it.
#     make -C oracle -f build_binary.mk build_binary
# Nothing from $(REF) is copied into tracked files; _ref/ is git-ignored.
include Makefile

build_binary: $(OUT)/build_binary

$(OUT)/build_binary: $(OBJ)/kenlm/lm/build_binary_main.o $(KENLM_OBJ)
	$(CXX) -o $@ $^ -lpthread

.PHONY: build_binary
