// rn_state.cuh -- checkpoint transpose of a sampler's chain state (rn_sampler_save / rn_sampler_restore, DESIGN.md 3.6).
//
// Between API calls a chain's whole state is the sampler's SoA arena, [field][element][chains] with the chain fastest, plus
// the tracked-diagnostics state, [201][n][chains] (rn_diag.cuh).  A checkpoint stores it chain-major -- one contiguous record
// per chain -- so that a range of chains is one byte range of the blob.  These two kernels move 32 chains x 32 record words
// per tile through shared memory: the SoA side is read (written) along the chain axis and the record side along the record,
// both coalesced.  Everything is moved as 32-bit words, so int, int64 and double fields take the same path and the bits are
// copied, never converted.
//
//   rn_k_state_pack    SoA chains [c0, c0 + count) -> records [count][rec_words] in a staging buffer
//   rn_k_state_unpack  records [count][rec_words]  -> SoA chains [c0, c0 + count)
//
// A field f occupies SoA words ptr_f[(e * C + c) * words_f + h] (element e < elems_f, h < words_f) and record words
// rec_word_f + e * words_f + h; fields are listed in increasing rec_word.  Compiled as a module of its own (rn_runtime.cpp:
// state_module), so the sampling modules do not change.  Also valid host C++ under RN_HOST_EMULATION, where one call of a
// kernel runs a whole CTA (the RN_ST_THREADS loops) and the barrier is a no-op.
#ifndef RN_STATE_CUH
#define RN_STATE_CUH

#define RN_STATE_MAX_FIELDS 32
#define RN_STATE_ROWS 8  // CTA = 32 x RN_STATE_ROWS threads; one tile = 32 chains x 32 record words

struct RnStateField {
  unsigned long long ptr;  // device address of the field's SoA array (word 0 of element 0, chain 0)
  long long elems;         // elements per chain
  int words;               // 32-bit words per element (1: int, 2: double / int64)
  int rec_word;            // first word of the field in a record
};

struct RnStateArgs {
  RnStateField f[RN_STATE_MAX_FIELDS];
  int n_fields;
  int pad0;
  long long rec_words;  // 32-bit words per record
  long long C;          // leading dimension (chains) of the SoA arrays
  long long c0;         // first SoA chain of this call
  long long count;      // chains of this call; record r <-> SoA chain c0 + r
  unsigned* staging;    // [count][rec_words]
};

#ifndef RN_STATE_ARGS_ONLY  // (the host runtime includes the argument block alone)
#ifdef RN_HOST_EMULATION
#define RN_ST_GLOBAL extern "C"
#define RN_ST_SHARED static thread_local
#define RN_ST_SYNC()
#define RN_ST_THREADS                                       \
  for (unsigned ty = 0; ty < RN_STATE_ROWS; ty++)           \
    for (unsigned tx = 0; tx < 32; tx++)
struct rn_st_dim3 { unsigned x, y, z; };
static thread_local rn_st_dim3 rn_st_block, rn_st_grid;
#define RN_ST_BLOCK rn_st_block
#define RN_ST_GRID rn_st_grid
#else
#define RN_ST_GLOBAL extern "C" __global__ __launch_bounds__(32 * RN_STATE_ROWS)
#define RN_ST_SHARED __shared__
#define RN_ST_SYNC() __syncthreads()
#define RN_ST_THREADS for (unsigned ty = threadIdx.y, tx = threadIdx.x, once_ = 0; once_ < 1; once_++)
#define RN_ST_BLOCK blockIdx
#define RN_ST_GRID gridDim
#endif

// record word w -> the SoA word of chain c holding it (fields sorted by rec_word; at most RN_STATE_MAX_FIELDS)
#ifdef RN_HOST_EMULATION
static inline
#else
__device__ __forceinline__
#endif
unsigned* rn_state_word(const RnStateArgs& a, long long w, long long c) {
  int f = 0;
  while (f + 1 < a.n_fields && a.f[f + 1].rec_word <= w) f++;
  const RnStateField& F = a.f[f];
  const long long k = w - F.rec_word, e = k / F.words, h = k - e * F.words;
  return (unsigned*)F.ptr + (e * a.C + c) * F.words + h;
}

// grid = (ceil(count / 32), tiles of record words, grid-stride over them)
RN_ST_GLOBAL void rn_k_state_pack(const RnStateArgs a) {
  RN_ST_SHARED unsigned tile[32][33];
  const long long ch0 = (long long)RN_ST_BLOCK.x * 32, wtiles = (a.rec_words + 31) / 32;
  for (long long wt = RN_ST_BLOCK.y; wt < wtiles; wt += RN_ST_GRID.y) {
    const long long w0 = wt * 32;
    RN_ST_THREADS {  // tile[word][chain] <- SoA: 32 consecutive chains of one word per row
      for (unsigned r = ty; r < 32; r += RN_STATE_ROWS)
        if (w0 + r < a.rec_words && ch0 + tx < a.count) tile[r][tx] = *rn_state_word(a, w0 + r, a.c0 + ch0 + tx);
    }
    RN_ST_SYNC();
    RN_ST_THREADS {  // records <- tile: 32 consecutive words of one chain per row
      for (unsigned r = ty; r < 32; r += RN_STATE_ROWS)
        if (ch0 + r < a.count && w0 + tx < a.rec_words) a.staging[(ch0 + r) * a.rec_words + w0 + tx] = tile[tx][r];
    }
    RN_ST_SYNC();
  }
}

RN_ST_GLOBAL void rn_k_state_unpack(const RnStateArgs a) {
  RN_ST_SHARED unsigned tile[32][33];
  const long long ch0 = (long long)RN_ST_BLOCK.x * 32, wtiles = (a.rec_words + 31) / 32;
  for (long long wt = RN_ST_BLOCK.y; wt < wtiles; wt += RN_ST_GRID.y) {
    const long long w0 = wt * 32;
    RN_ST_THREADS {  // tile[chain][word] <- records
      for (unsigned r = ty; r < 32; r += RN_STATE_ROWS)
        if (ch0 + r < a.count && w0 + tx < a.rec_words) tile[r][tx] = a.staging[(ch0 + r) * a.rec_words + w0 + tx];
    }
    RN_ST_SYNC();
    RN_ST_THREADS {  // SoA <- tile
      for (unsigned r = ty; r < 32; r += RN_STATE_ROWS)
        if (w0 + r < a.rec_words && ch0 + tx < a.count) *rn_state_word(a, w0 + r, a.c0 + ch0 + tx) = tile[tx][r];
    }
    RN_ST_SYNC();
  }
}
#endif  // RN_STATE_ARGS_ONLY
#endif  // RN_STATE_CUH
