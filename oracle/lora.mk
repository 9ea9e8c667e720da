# oracle/lora.mk -- TEST INFRASTRUCTURE, not product code.
#
# Builds oracle/_ref/lora_merge (lora_merge.cpp): llama.cpp's llama_model_apply_lora_from_file run on a full GGJT model,
# the merged model written back out.  lora_merge.cpp includes the reference's vendor/llama.cpp/llama.cpp where it lies
# (never copied into this repo) and links Makefile's ggml.o and k_quants.o, so the merge runs the same arithmetic as the
# other reference binaries.  Only built where $(REF) exists; the GPU box uses the prebuilt file that travels with the
# snapshot.
#
#     make -C oracle -f lora.mk lora_merge

include Makefile

.PHONY: lora_merge
ifneq ($(wildcard $(LL)/llama.cpp),)
lora_merge: $(OUT)/lora_merge
else
lora_merge:
	@echo "oracle: $(REF) absent -- using prebuilt oracle/_ref/lora_merge (if any)"
endif

$(OUT)/lora_merge: lora_merge.cpp $(LL)/llama.cpp $(OUT)/ggml.o $(OUT)/k_quants.o
	g++ $(CXXFLAGS) -DLLAMA_CPP_PATH='"$(LL)/llama.cpp"' lora_merge.cpp $(OUT)/ggml.o $(OUT)/k_quants.o -o $@
