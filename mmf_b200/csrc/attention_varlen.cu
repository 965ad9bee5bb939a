// Packed (variable-length) self-attention entry points: the VARLEN instantiations of the kernels in attention.cu,
// compiled in their own translation unit so that the dense kernels keep their code (see the note above attn_fwd).
#define MMFB_ATTN_VARLEN_TU
#include "attention.cu"
