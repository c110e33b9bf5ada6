/* C ABI of the tensor-core GEMM of libmia_scan.so (sm_90a: wgmma.mma_async + TMA tensor-map loads).
 *
 *   C[M, N] = act( A[M, K] . W[N, K]^T + bias[N] )
 *
 * It replaces the library GEMMs (cuBLAS through nn.Linear / torch.einsum, cuDNN through kernel==stride nn.Conv2d) on the
 * projections of the hot path:
 *   SS2D      in_proj / out_proj / x_proj   R2GenCSR/VMamba/classification/models/vmamba.py:751, 775, 386
 *   Mamba     in_proj / x_proj / out_proj   CXPMRG_Bench_MambaXray_VL/arm/Finetuning/mamba_simple.py:408-414, 686, 708
 *   SmallPatchEmbed conv 16/16, 4/4, 1x1    HD_Xray_Pretrain_MAE/pretrain/patch_embed.py:25-41 (one GEMM each over patches)
 *   timm Block qkv / proj / fc1 / fc2       HD_Xray_Pretrain_MAE/pretrain/models/mae.py:64-66, 82-84
 *
 * A (M x K, row pitch lda) and W (N x K, row pitch ldw: nn.Linear's weight layout) hold bf16 or fp16 with K contiguous;
 * accumulation is fp32 in tensor memory; bias is fp32 (may be NULL); C (row pitch ldc) is written in the input dtype or in
 * fp32.  Device pointers only, 16-byte aligned A and W, lda / ldw multiples of 8 elements; any M, N; K % 8 == 0 is implied
 * by the pitch rule (a K tail inside the last 64-wide block is zero-filled by TMA).  Asynchronous on `cuda_stream`.
 * Returns 0 or a negative MIA_GEMM_E* code; mia_gemm_last_error() holds the message (thread-local).
 */
#ifndef MIA_GEMM_H_
#define MIA_GEMM_H_

#ifdef __cplusplus
extern "C" {
#endif

enum { MIA_GEMM_F32 = 0, MIA_GEMM_F16 = 1, MIA_GEMM_BF16 = 2 };          /* same numbering as MIA_F32 / MIA_F16 / MIA_BF16 */
enum { MIA_ACT_NONE = 0, MIA_ACT_RELU = 1, MIA_ACT_GELU = 2, MIA_ACT_SILU = 3 };   /* GELU: exact (erf) form, nn.GELU() default */
enum { MIA_GEMM_OK = 0, MIA_GEMM_EINVAL = -1, MIA_GEMM_ECUDA = -2 };

int mia_gemm_tn(const void *A, const void *W, const float *bias, void *C, int M, int N, int K, long long lda, long long ldw,
                long long ldc, int in_dtype, int out_dtype, int act, void *cuda_stream);
/* General form: each operand may also be stored with its M / N index contiguous ("MN-major"), which is what the two
 * backward contractions of a linear layer need with NO transposed copies:
 *   a_mn_major = 0: A is [M][K] (pitch lda)      a_mn_major = 1: A is stored [K][M] (pitch lda), i.e. A^T read in place
 *   b_mn_major = 0: B is [N][K] (pitch ldb)      b_mn_major = 1: B is stored [K][N] (pitch ldb)
 *   dX[tok, in]  = dY[tok, out] . W[out, in]      -> A = dY (0),            B = W stored [K = out][N = in]   (1)
 *   dW[out, in]  = dY[tok, out]^T . X[tok, in]    -> A = dY stored [K][M] (1), B = X stored [K = tok][N = in] (1)
 * The wgmma transpose bits select the layout; TMA boxes are [64 k][64 mn] for it. */
int mia_gemm(const void *A, const void *B, const float *bias, void *C, int M, int N, int K, long long lda, long long ldb, long long ldc,
             int a_mn_major, int b_mn_major, int in_dtype, int out_dtype, int act, void *cuda_stream);
/* SwiGLU MLP (w3(silu(w1(x)) * w2(x)), models_mamba.py:59-83) around the same kernel.  Hp = H rounded up to a multiple of 64.
 *
 * Forward: one GEMM whose B tile pairs W1 and W2 rows: a = x W1^T + b1 and b = x W2^T + b2 accumulate in fp32 in the same
 * thread, and the epilogue rounds a and b to dtype (bit-identical to two mia_gemm_tn calls with those biases) and writes
 *   h (M, H, pitch ldh)      round(silu(a) * b), computed from the rounded a and b
 *   ab (M, 2 Hp, pitch ldab) a in columns [0, H), b in [Hp, Hp + H), pad columns 0; NULL (inference) writes h only.
 * x (M, K), w1 / w2 (H, K) nn.Linear layout; b1 / b2 fp32 (H) or NULL.
 *
 * Backward: g = dy . W3 (dy (M, N_out), W3 (N_out, H) read in place), and from a, b in ab and s = sigmoid(a):
 *   dab (M, 2 Hp, pitch lddab)  da = g b s (1 + a (1 - s)) in [0, H), db = g a s in [Hp, Hp + H), each rounded once, pads 0
 *   h (M, H, pitch ldh)         round(a s b), bit-identical to the forward's h, for W3's gradient (NULL: not written).
 *
 * dtype is MIA_GEMM_BF16 or MIA_GEMM_F16 for every operand.  Pitches are multiples of 8 elements covering a row (ldab /
 * lddab >= 2 Hp), pointers 16-byte aligned.  Errors as for mia_gemm_tn. */
int mia_gemm_swiglu_fwd(const void *x, const void *w1, const void *w2, const float *b1, const float *b2, void *h, void *ab, int M, int H,
                        int K, long long ldx, long long ldw1, long long ldw2, long long ldh, long long ldab, int dtype, void *cuda_stream);
int mia_gemm_swiglu_bwd(const void *dy, const void *w3, const void *ab, void *dab, void *h, int M, int H, int N_out, long long lddy,
                        long long ldw3, long long ldab, long long lddab, long long ldh, int dtype, void *cuda_stream);
/* GELU MLP (fc2(gelu(fc1(x))), vmamba.py:495-514 and timm's Mlp) around the same kernel.  Hp = H rounded up to a multiple of 8.
 *
 * Forward: fc1 as one GEMM, x (M, K), w1 (H, K) nn.Linear layout, b1 fp32 (H) or NULL.  The epilogue writes
 *   pre (M, H, pitch ldpre)  round(x W1^T + b1), bit-identical to mia_gemm_tn(x, w1, b1) (same k order, fp32 bias add)
 *   h (M, H, pitch ldh)      round(0.5 p (1 + erf(p / sqrt 2))) in fp32 from the rounded p = pre: F.gelu(pre)
 * and 0 in columns [H, Hp) of both; pre NULL (inference) writes h only.
 *
 * Backward: g = dy . W2 in fp32, never rounded (dy (M, N_out), W2 (N_out, H) read in place), and from p in pre:
 *   dpre (M, H, pitch lddpre)  round(g (Phi(p) + p phi(p))), Phi from erfc, recomputed in fp64 where the factor is below
 *                              2^-8 (around its root at p = -0.7518); 0 in columns [H, Hp)
 *   h (M, H, pitch ldh)        the forward's expression, bit-identical to its h, for W2's gradient (NULL: not written).
 *
 * dtype is MIA_GEMM_BF16 or MIA_GEMM_F16 for every operand.  Pitches are multiples of 8 elements covering a row (so
 * ldpre, lddpre, ldh >= Hp), pointers 16-byte aligned.  Errors as for mia_gemm_tn. */
int mia_gemm_gelu_fwd(const void *x, const void *w1, const float *b1, void *h, void *pre, int M, int H, int K, long long ldx, long long ldw1,
                      long long ldh, long long ldpre, int dtype, void *cuda_stream);
int mia_gemm_gelu_bwd(const void *dy, const void *w2, const void *pre, void *dpre, void *h, int M, int H, int N_out, long long lddy,
                      long long ldw2, long long ldpre, long long lddpre, long long ldh, int dtype, void *cuda_stream);
/* ViT-MAE attention (timm Attention: softmax(q k^T dh^-0.5) v per image and head, no mask, no dropout) on wgmma + TMA.
 * C = H dh.  qkv is the qkv GEMM's output read in place: (B, N, 3, H, dh), row pitch ld_qkv >= 3C, q / k / v of head h in
 * columns h dh, C + h dh, 2C + h dh.  Rows past token N - 1 of an image are never read as keys or written.
 *
 * Forward: o (B, N, C, pitch ld_o >= C) token-major, the layout the proj GEMM consumes; P is rounded to dtype before P V
 * and O / l once.  lse (B, H, N) fp32 = logsumexp of the scaled logits per query row; NULL (inference) writes none.
 *
 * Backward: from dout = dL/do (B, N, C, pitch ld_do) writes dq / dk / dv straight into the packed dqkv (B, N, 3C, pitch
 * ld_dqkv), the layout of qkv, i.e. the qkv GEMM's output gradient.  delta (B, H, N) fp32 is caller-owned scratch
 * (rowsum(dout o o)).  Two launches (dq, then dk / dv), no atomics: the results are bit-reproducible.
 *
 * dh is 32, 64 or 80; B, N, H >= 1; dtype MIA_GEMM_BF16 or MIA_GEMM_F16 for every 16-bit operand; pitches multiples of 8
 * elements covering a row; pointers 16-byte aligned.  Errors as for mia_gemm_tn. */
int mia_attn_fwd(const void *qkv, void *o, float *lse, int B, int N, int H, int dh, long long ld_qkv, long long ld_o, int dtype, void *cuda_stream);
int mia_attn_bwd(const void *qkv, const void *o, const void *dout, const float *lse, float *delta, void *dqkv, int B, int N, int H, int dh,
                 long long ld_qkv, long long ld_o, long long ld_do, long long ld_dqkv, int dtype, void *cuda_stream);
/* Segment-causal cross-attention (the ARM pre-training decoder's CrossAttention: softmax(q k^T dh^-0.5 + mask) v with
 * mask 0 where key // seg <= query // seg and -inf elsewhere) on the kernels above.  C = H dh, dh = 64.  q is the q GEMM's
 * output (B, N, C, pitch ld_q >= C), kv the kv GEMM's output (B, N, 2C, pitch ld_kv >= 2C) with k / v of head h in columns
 * h dh / C + h dh; both are read in place.  Key tiles that no query of a tile can see are skipped.
 *
 * Forward: o and lse as for mia_attn_fwd (lse NULL: inference).  Backward: dq into (B, N, C, pitch ld_dq >= C) and dk / dv
 * into the packed (B, N, 2C, pitch ld_dkv >= 2C): the output gradients of the q and kv GEMMs.  delta (B, H, N) fp32 is
 * caller-owned scratch.  No atomics: the results are bit-reproducible.
 *
 * 1 <= B, H <= 65535; N >= 1; 1 <= seg <= N; dtype MIA_GEMM_BF16 or MIA_GEMM_F16; pitches multiples of 8 elements covering
 * a row; pointers 16-byte aligned.  Errors as for mia_gemm_tn. */
int mia_xattn_fwd(const void *q, const void *kv, void *o, float *lse, int B, int N, int H, int dh, int seg, long long ld_q, long long ld_kv,
                  long long ld_o, int dtype, void *cuda_stream);
int mia_xattn_bwd(const void *q, const void *kv, const void *o, const void *dout, const float *lse, float *delta, void *dq, void *dkv, int B, int N,
                  int H, int dh, int seg, long long ld_q, long long ld_kv, long long ld_o, long long ld_do, long long ld_dq, long long ld_dkv, int dtype,
                  void *cuda_stream);
const char *mia_gemm_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* MIA_GEMM_H_ */
