// jf_matrix.hpp -- GF(2) rectangular matrix used as the k-mer hash.
//
// Behavioural contract (reference include/jellyfish/rectangular_binary_matrix.hpp):
//  * r x c bits, r <= 64, stored one uint64 per column                      (:30-38)
//  * times(v) = XOR of columns[c-1-i] over the set bits i of the 2k-bit key (:223-261):
//    the column index is REVERSED with respect to the bit index.
//  * identity (no columns) when the table is as large as the key space: v & mask (:225)
//  * the hash matrix of a table is the pseudo-inverse of a freshly drawn random
//    matrix (lib/rectangular_binary_matrix.cc:160-210,240-247; large_hash_array.hpp:992-1002)
// Own implementation written against that contract (the inverse is a row-wise Gauss-Jordan, see pseudo_inverse).
#ifndef JFB_MATRIX_HPP
#define JFB_MATRIX_HPP
#include <stdint.h>
#include <vector>
#include <stdexcept>
#include <algorithm>
#include "jf_random.hpp"

namespace jfb {

class gf2_matrix {
  unsigned r_, c_;
  bool     identity_;            // "no columns" identity of the reference (r == c)
  std::vector<uint64_t> col_;    // c_ columns, bit j of col_[i] = row j (row 0 = LSB of the result)

  uint64_t cmask() const { return r_ >= 64 ? ~(uint64_t)0 : (((uint64_t)1 << r_) - 1); }
public:
  gf2_matrix() : r_(0), c_(0), identity_(true) { }
  gf2_matrix(unsigned r, unsigned c) : r_(r), c_(c), identity_(false), col_(c, 0) {
    if(r == 0 || r > 64 || c == 0 || c > 256) throw std::out_of_range("Invalid matrix size");
  }
  template<typename It>
  gf2_matrix(unsigned r, unsigned c, It raw) : r_(r), c_(c), identity_(false), col_(c, 0) {
    for(unsigned i = 0; i < c; ++i, ++raw) col_[i] = (uint64_t)*raw & cmask();
  }
  static gf2_matrix identity(unsigned c) { gf2_matrix m; m.r_ = m.c_ = c; m.identity_ = true; return m; }
  // the "low identity" r x c matrix: picks the low r bits of the vector
  static gf2_matrix low_identity(unsigned r, unsigned c) {
    gf2_matrix m(r, c);
    unsigned row = std::min(r, c), col = c - row;
    for(unsigned i = col; i < c; ++i) m.col_[i] = (uint64_t)1 << (row - 1 - (i - col));
    return m;
  }

  unsigned r() const { return r_; }
  unsigned c() const { return c_; }
  bool is_identity() const { return identity_; }
  uint64_t operator[](unsigned i) const { return identity_ ? ((uint64_t)1 << i) : col_[i]; }
  const std::vector<uint64_t>& columns() const { return col_; }
  unsigned nb_words() const { return (c_ + 63) / 64; }

  bool is_low_identity() const {
    if(identity_) return true;
    unsigned row = std::min(r_, c_), col = c_ - row;
    for(unsigned i = 0; i < col; ++i) if(col_[i]) return false;
    for(unsigned i = col; i < c_; ++i) if(col_[i] != ((uint64_t)1 << (row - 1 - (i - col)))) return false;
    return true;
  }

  bool operator==(const gf2_matrix& o) const {
    if(r_ != o.r_ || c_ != o.c_ || identity_ != o.identity_) return false;
    return identity_ || col_ == o.col_;
  }
  bool operator!=(const gf2_matrix& o) const { return !(*this == o); }

  // v: little-endian array of nb_words() 64-bit words holding the c-bit vector.
  uint64_t times(const uint64_t* v) const {
    if(identity_) return v[0] & cmask();
    uint64_t res = 0;
    for(unsigned i = 0; i < c_; ++i)
      if((v[i >> 6] >> (i & 63)) & 1) res ^= col_[c_ - 1 - i];
    return res;
  }

  void randomize(glibc_random& rng) {
    for(unsigned i = 0; i < c_; ++i) col_[i] = rng.bits(64) & cmask();
  }

  // Pseudo-inverse.  Split the key v into its low s = min(r, c) bits vl and the rest vh, and the matrix
  // accordingly: M v = Ml vl ^ Mh vh with Ml square (s x s).  The hash position w = M v together with the
  // explicit high bits vh determines the key: vl = Ml^-1 (w ^ Mh vh).  The result is the matrix
  // N = Ml^-1 [Mh | I] acting on y = [vh : w] (w in the low s bits, vh above them), i.e. N y = vl -- what the
  // reference calls pseudo_inverse (it inverts the square matrix obtained by stacking an identity for vh on
  // top of M and keeps the bottom rows; the inverse being unique, any elimination order gives the same N).
  // Here: Gauss-Jordan on ROWS of the augmented system (Ml | Mh | I).  Throws std::domain_error when Ml is singular.
  gf2_matrix pseudo_inverse() const {
    if(identity_) return *this;
    const unsigned s = std::min(r_, c_);
    struct eq { uint64_t lo; uint64_t hi[4]; uint64_t w; };      // coefficients on vl, on vh (c - s < 256 bits), on w
    std::vector<eq> R(s);
    for(unsigned j = 0; j < s; ++j) {
      eq q = { 0, { 0, 0, 0, 0 }, (uint64_t)1 << j };
      for(unsigned i = 0; i < c_; ++i) {
        const uint64_t bit = (col_[c_ - 1 - i] >> j) & 1;          // key bit i feeds column c-1-i
        if(i < s) q.lo |= bit << i;
        else q.hi[(i - s) >> 6] |= bit << ((i - s) & 63);
      }
      R[j] = q;
    }
    for(unsigned p = 0; p < s; ++p) {
      unsigned q = p;
      while(q < s && !((R[q].lo >> p) & 1)) ++q;
      if(q == s) throw std::domain_error("hash matrix has no pseudo-inverse");
      std::swap(R[p], R[q]);
      for(unsigned t = 0; t < s; ++t)
        if(t != p && ((R[t].lo >> p) & 1)) { R[t].lo ^= R[p].lo; for(int h = 0; h < 4; ++h) R[t].hi[h] ^= R[p].hi[h]; R[t].w ^= R[p].w; }
    }
    // row p now reads  vl_p = hi . vh ^ w . (M v)
    gf2_matrix res(r_, c_);
    for(unsigned p = 0; p < s; ++p)
      for(unsigned t = 0; t < c_; ++t) {
        const uint64_t coef = t < s ? (R[p].w >> t) & 1 : (R[p].hi[(t - s) >> 6] >> ((t - s) & 63)) & 1;
        if(coef) res.col_[c_ - 1 - t] |= (uint64_t)1 << p;
      }
    return res;
  }

  // Redraw until pseudo-invertible, return the pseudo-inverse (the table's hash matrix).
  gf2_matrix randomize_pseudo_inverse(glibc_random& rng) {
    for(;;) {
      randomize(rng);
      try { return pseudo_inverse(); } catch(std::domain_error&) { }
    }
  }
};

} // namespace jfb
#endif
