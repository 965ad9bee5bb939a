// Dense self-attention with a causal tail (causal_len > 0): the CAUSAL instantiations of the kernels in attention.cu,
// compiled in their own translation unit so that the dense kernels keep their code (see the note above attn_fwd).
#define MMFB_ATTN_CAUSAL_TU
#include "attention.cu"
