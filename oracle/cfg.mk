# oracle/cfg.mk -- TEST INFRASTRUCTURE, not product code.
#
# Builds two things under oracle/_ref/:
#   main      llama.cpp's `main` program, compiled from the reference's vendor/llama.cpp/examples/main/main.cpp where it
#             lies, as vendor/llama.cpp/Makefile's `main` target does (tests/golden/gen_golden_cfg.py runs it with
#             --cfg-negative-prompt);
#   cfg_shim  (cfg_shim.cpp): llama.cpp's llama_sample_classifier_free_guidance run on given rows of logits.  cfg_shim.cpp includes the reference's vendor/llama.cpp/llama.cpp where it lies (never copied into this repo)
# and links Makefile's ggml.o and k_quants.o with Makefile's flags, so the guidance arithmetic is compiled as the
# reference build compiles it (the same FMA contractions).  Only built where $(REF) exists; elsewhere the prebuilt file,
# if any, is used.
#
#     make -C oracle -f cfg.mk cfg

include Makefile

.PHONY: cfg
ifneq ($(wildcard $(LL)/examples/main/main.cpp),)
cfg: $(OUT)/cfg_shim $(OUT)/main
else
cfg:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/cfg_shim and main (if any)"
endif

$(OUT)/main: $(LL)/examples/main/main.cpp $(OUT)/ggml.o $(OUT)/llama.o $(OUT)/common.o $(OUT)/k_quants.o
	g++ $(CXXFLAGS) $^ -o $@

$(OUT)/cfg_shim: cfg_shim.cpp $(LL)/llama.cpp $(OUT)/ggml.o $(OUT)/k_quants.o
	g++ $(CXXFLAGS) -DLLAMA_CPP_PATH='"$(LL)/llama.cpp"' cfg_shim.cpp $(OUT)/ggml.o $(OUT)/k_quants.o -o $@
