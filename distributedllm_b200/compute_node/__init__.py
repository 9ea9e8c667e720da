"""Compute node: holds ONE model slice on one H100 and answers the reference's RPC (status, upload, load_slice,
propagate_forward, clear_context).  Mirrors distllm/compute_node/* of the reference; the per-slice forward runs on
the GPU through the `llm` module (distributedllm_b200/csrc/llm_module.cpp -> libb200slice.so)."""
