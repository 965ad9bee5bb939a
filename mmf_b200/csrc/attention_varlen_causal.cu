// Packed (variable-length) self-attention with a causal tail (causal_len > 0): the VARLEN && CAUSAL instantiations of the
// kernels in attention.cu, compiled in their own translation unit so that the other kernels keep their code (see the
// note above attn_fwd).
#define MMFB_ATTN_VARLEN_CAUSAL_TU
#include "attention.cu"
