// oracle/cfg_shim.cpp -- TEST INFRASTRUCTURE, not product code.
//
// Runs llama.cpp's own llama_sample_classifier_free_guidance on given rows of logits.  The vendored llama.cpp translation
// unit is #included where it lies (LLAMA_CPP_PATH), as lora_merge.cpp does, so the shim can fill a context's logits.  It
// loads a full GGJT model (only for its n_vocab), makes a session context and a guidance context, and for each row pair
// puts the base row into the candidates and the guidance row into the guidance context's logits, calls the real function,
// and writes the candidates' logits out.
//
//     cfg_shim MODEL ROWS OUT SCALE SMOOTH_FACTOR
//
// ROWS holds n pairs of float32 rows: all n base rows, then all n guidance rows (n = file size / (8 * n_vocab)).  OUT gets
// the n guided rows.
#include LLAMA_CPP_PATH

#include <cstdio>

int main(int argc, char ** argv) {
    if (argc < 6) {
        fprintf(stderr, "usage: %s MODEL ROWS OUT SCALE SMOOTH_FACTOR\n", argv[0]);
        return 2;
    }
    const float scale = strtof(argv[4], nullptr), sf = strtof(argv[5], nullptr);
    llama_context_params params = llama_context_default_params();
    params.n_ctx = 8;
    llama_model * model = llama_load_model_from_file(argv[1], params);
    if (!model) return 1;
    llama_context * ctx = llama_new_context_with_model(model, params);
    llama_context * gctx = llama_new_context_with_model(model, params);
    if (!ctx || !gctx) return 1;
    const int n_vocab = llama_n_vocab(ctx);
    FILE * fi = fopen(argv[2], "rb");
    if (!fi) return 1;
    std::vector<float> rows;
    fseek(fi, 0, SEEK_END); rows.resize((size_t) ftell(fi) / 4); fseek(fi, 0, SEEK_SET);
    if (fread(rows.data(), 4, rows.size(), fi) != rows.size()) return 1;
    fclose(fi);
    const size_t n = rows.size() / (2 * (size_t) n_vocab);
    std::vector<float> out(n * n_vocab);
    std::vector<llama_token_data> cand(n_vocab);
    for (size_t k = 0; k < n; k++) {
        const float * b = rows.data() + k * n_vocab, * g = rows.data() + (n + k) * n_vocab;
        for (int i = 0; i < n_vocab; i++) cand[i] = llama_token_data{i, b[i], 0.0f};
        llama_token_data_array arr{cand.data(), cand.size(), false};
        gctx->logits.assign(g, g + n_vocab);
        llama_sample_classifier_free_guidance(ctx, &arr, gctx, scale, sf);
        for (int i = 0; i < n_vocab; i++) out[k * n_vocab + i] = cand[i].logit;
    }
    FILE * fo = fopen(argv[3], "wb");
    if (!fo || fwrite(out.data(), 4, out.size(), fo) != out.size()) return 1;
    fclose(fo);
    llama_free(gctx);
    llama_free(ctx);
    llama_free_model(model);
    return 0;
}
