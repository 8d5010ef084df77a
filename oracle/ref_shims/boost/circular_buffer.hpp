// boost/circular_buffer.hpp stand-in: the members FailureDetector uses (recovery_behaviors.h), backed by a deque.
// push_back into a full buffer drops the front element, and a buffer of capacity 0 takes nothing, as boost's does.
#ifndef REF_SHIM_BOOST_CIRCULAR_BUFFER
#define REF_SHIM_BOOST_CIRCULAR_BUFFER
#include <cstddef>
#include <deque>
namespace boost {
template <typename T> class circular_buffer {
 public:
  typedef std::size_t size_type;
  void set_capacity(size_type c) {
    cap_ = c;
    while (d_.size() > cap_) d_.pop_back();   // boost removes the last elements
  }
  void push_back(const T& v) {
    if (cap_ == 0) return;
    if (d_.size() == cap_) d_.pop_front();
    d_.push_back(v);
  }
  size_type size() const { return d_.size(); }
  size_type capacity() const { return cap_; }
  const T& operator[](size_type i) const { return d_[i]; }
  T& operator[](size_type i) { return d_[i]; }
  void clear() { d_.clear(); }

 private:
  std::deque<T> d_;
  size_type cap_ = 0;
};
}  // namespace boost
#endif
