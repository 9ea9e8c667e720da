# oracle/perplexity.mk -- TEST INFRASTRUCTURE, not product code.
#
# Builds oracle/_ref/perplexity: llama.cpp's `perplexity` program, compiled from the reference's
# vendor/llama.cpp/examples/perplexity/perplexity.cpp where it lies (never copied into this repo), as
# vendor/llama.cpp/Makefile's `perplexity` target does.  b200_perplexity_windows reproduces what it prints.
# It reuses Makefile's flags and object rules (ggml.o, llama.o, common.o, k_quants.o), so the program runs the
# same arithmetic as the other reference binaries.  Only built where $(REF) exists; the GPU box uses the
# prebuilt file that travels with the snapshot.
#
#     make -C oracle -f perplexity.mk perplexity

include Makefile

.PHONY: perplexity
ifneq ($(wildcard $(LL)/examples/perplexity/perplexity.cpp),)
perplexity: $(OUT)/perplexity
else
perplexity:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/perplexity (if any)"
endif

$(OUT)/perplexity: $(LL)/examples/perplexity/perplexity.cpp $(OUT)/ggml.o $(OUT)/llama.o $(OUT)/common.o $(OUT)/k_quants.o
	g++ $(CXXFLAGS) $^ -o $@
