# Builds _ref/libteb_ref_recovery.so (test infrastructure): the reference's own recovery_behaviors.cpp (FailureDetector)
# compiled where it lies against the stand-in headers in ref_shims/ (boost::circular_buffer, ROS message types, g2o's
# misc helpers), with the driver ref_recovery_driver.cpp. Only possible where the reference sources exist; outputs only
# into _ref/. Used by tests/test_reference_pin_recovery.py:  make -C oracle -f ref_recovery.mk
REF ?= /root/reference
REF_SHIMS = $(shell find ref_shims -type f)
all: _ref/libteb_ref_recovery.so
_ref/libteb_ref_recovery.so: ref_recovery_driver.cpp $(REF_SHIMS)
	@mkdir -p _ref
	g++ -std=c++14 -O2 -ffp-contract=off -fPIC -shared -w -Iref_shims -I$(REF)/include -o $@ ref_recovery_driver.cpp \
	    $(REF)/src/recovery_behaviors.cpp
clean:
	rm -f _ref/libteb_ref_recovery.so
