// oracle/lora_merge.cpp -- TEST INFRASTRUCTURE, not product code.
//
// Merges a LoRA adapter into a full GGJT model with llama.cpp's own code and writes the merged model back out.  The
// vendored llama.cpp translation unit is #included where it lies (LLAMA_CPP_PATH), as ref_shim.cpp includes
// tensor_processor.cpp, so the tool can read the loaded model's tensors.  It loads the model with use_mmap = false (main
// disables mmap under --lora), calls the real llama_model_apply_lora_from_file(model, lora, base, n_threads), and copies
// the input file with every tensor's bytes replaced by the merged ones.  slice_model then cuts merged slices.
//
//     lora_merge MODEL ADAPTER BASE|- OUT [N_THREADS]
//
// Prints the merge's wall time in ms on stdout ("merge_ms <t>").
#include LLAMA_CPP_PATH

#include <chrono>
#include <cstdio>

int main(int argc, char ** argv) {
    if (argc < 5) {
        fprintf(stderr, "usage: %s MODEL ADAPTER BASE|- OUT [N_THREADS]\n", argv[0]);
        return 2;
    }
    const char * base = strcmp(argv[3], "-") == 0 ? nullptr : argv[3];
    const int n_threads = argc > 5 ? atoi(argv[5]) : 4;
    llama_context_params params = llama_context_default_params();
    params.use_mmap = false;
    llama_model * model = llama_load_model_from_file(argv[1], params);
    if (!model) return 1;
    const auto t0 = std::chrono::steady_clock::now();
    if (llama_model_apply_lora_from_file(model, argv[2], base, n_threads) != 0) return 1;
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();

    // the input file, tensor records walked as llama_file_loader reads them (GGJT v3, seven hparams)
    FILE * fi = fopen(argv[1], "rb");
    if (!fi) return 1;
    std::vector<uint8_t> buf;
    fseek(fi, 0, SEEK_END); buf.resize((size_t) ftell(fi)); fseek(fi, 0, SEEK_SET);
    if (fread(buf.data(), 1, buf.size(), fi) != buf.size()) return 1;
    fclose(fi);
    size_t pos = 0;
    auto u32 = [&]() { uint32_t v; memcpy(&v, buf.data() + pos, 4); pos += 4; return v; };
    u32(); u32();
    const uint32_t n_vocab = u32();
    for (int i = 0; i < 6; i++) u32();
    for (uint32_t i = 0; i < n_vocab; i++) { const uint32_t len = u32(); pos += len + 4; }
    std::unordered_map<std::string, ggml_tensor *> by_name(model->tensors_by_name.begin(), model->tensors_by_name.end());
    while (pos < buf.size()) {
        const uint32_t n_dims = u32(), name_len = u32();
        u32();
        pos += 4 * n_dims;
        const std::string name((const char *) buf.data() + pos, name_len);
        pos = (pos + name_len + 31) & ~(size_t) 31;
        ggml_tensor * t = by_name.at(name);
        memcpy(buf.data() + pos, t->data, ggml_nbytes(t));
        pos += ggml_nbytes(t);
    }
    FILE * fo = fopen(argv[4], "wb");
    if (!fo || fwrite(buf.data(), 1, buf.size(), fo) != buf.size() || fclose(fo) != 0) return 1;
    llama_free_model(model);
    printf("merge_ms %.3f\n", ms);
    return 0;
}
