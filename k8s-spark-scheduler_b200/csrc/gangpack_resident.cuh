// gangpack_resident.cuh -- private to libgangpack: the update protocol the five resident tables share (reservation, overhead,
// label, node and driver table).  Each table keeps its own columns, Delta, checks, kernels and refusals in its .cu file.
//
// A table is live from a successful reset until a CUDA error breaks it; every reader checks need() first.
//   reset        the columns laid out (take_cols) and filled by the table, one synchronise, then live with seq = 0
//   update       the table's host checks, the delta staged on the context's call buffer with a zeroed status word and
//                checked while the table is still live (a staging error changes nothing), then begin(): live = false and
//                ++seq; the table's kernels, of which only the check writes before the error word is complete, and only the
//                stamps; then commit(): one synchronise, live = true and the refusal decoded from the word
// An empty delta goes through the same steps: it is accepted and changes no row.
//
// The stamps are the last pieces of every take_cols layout, zeroed by the reset.  An update's check stamps each entry it
// writes with the update's number seq (stamped_twice): an entry written twice by one delta finds seq there already.  When seq
// wraps to 0 the stamps are zeroed first and seq restarts at 1, so no stamp left from an earlier update equals a later one.
//
// Included by gangpack_ctx.cuh before gp_ctx, which holds the tables: the helpers take the context as the parameter Ctx.
#pragma once

#include <algorithm>
#include <cstdint>

template <class Size>
struct ResidentTable {
    const char* absent;                       // the readers' refusal when the table is not live: "no X table (gp_X_table_reset first)"
    bool live = false;                        // reset and not broken by a CUDA error since
    Size size{};
    DevBuf cols;                              // the columns, the stamps last, in one block
    uint32_t seq = 0;                         // the last update's stamp

    explicit ResidentTable(const char* absent) : absent(absent) {}

    Need need() const { return live ? Need{GP_OK, nullptr} : Need{GP_ERR_INVALID, absent}; }

    // fill(a) lays out the columns of z on a (take_cols), reserves and fills them, and returns the status of anything else it
    // stages
    template <class Ctx, class Fill> gp_status reset(Ctx* c, const Size& z, Fill&& fill) {
        live = false;
        GP_CUDA(c, cudaSetDevice(c->device));
        Arena a{cols, c->stream};
        GP_TRY(fill(a));
        GP_TRY(a.sync(c));
        size = z;
        seq = 0;
        live = true;
        return GP_OK;
    }

    // After the delta's staging was checked: from here on the table's own buffers are written, and a CUDA error leaves no
    // table (reset and replay).  tc holds the table's take_cols layout; the stamps are first_stamp .. last_stamp.
    template <class Ctx, class A, class B> gp_status begin(Ctx* c, Arena& tc, Piece<A> first_stamp, Piece<B> last_stamp) {
        live = false;
        if (++seq == 0) {
            tc.fill(first_stamp, last_stamp, 0);
            seq = 1;
        }
        return tc.check(c);
    }

    // After the table's kernels: the status word read into *hw, one synchronise, the table live again, and the first refusal
    // of `table` whose bits the word carries
    template <class Ctx, class Word, size_t K>
    gp_status commit(Ctx* c, Arena& ar, Piece<Word> word, Word* hw, const Refusal (&table)[K], const char* who) {
        GP_CUDA(c, cudaGetLastError());
        ar.get(hw, word);
        GP_TRY(ar.sync(c));
        live = true;
        return refuse(c, refusal_bits(*hw), table, who);
    }

private:
    static int refusal_bits(int w) { return w; }
    template <class Word> static int refusal_bits(const Word& w) { return w.err; }
};

// The grid of an update's grid-stride kernels over n items of `threads` threads: at least one block, at most 8 per SM
static inline unsigned update_grid(long long n, int threads, int sm_count) {
    return (unsigned)std::max<long long>(1, std::min<long long>((n + threads - 1) / threads, (long long)sm_count * 8));
}

// An update's check stamps the entry it writes: true when this update stamped it already (the entry is given twice)
__device__ __forceinline__ bool stamped_twice(uint32_t* stamp, uint32_t seq) { return atomicExch(stamp, seq) == seq; }
