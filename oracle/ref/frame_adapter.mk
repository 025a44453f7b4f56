# TEST INFRASTRUCTURE ONLY.  The product's FrameConstructor (include/pslam_reference_adapter.hpp) compiled against the reference's headers, over the reference's
# Frame of libmatch_ref.so and the CUDA library, with the plain-array entry points of ref/frame_adapter_driver.cc (tests/test_frame_adapter_gpu.py).
# Run from oracle/ as  make -f ref/frame_adapter.mk frame-adapter  (called by __graft_entry__.build() next to `make adapter`); the variables and the
# libmatch_ref.so recipe are the ones of oracle/Makefile.
include Makefile

_ref/libframe_adapter_ref.so: ref/frame_adapter_driver.cc ../include/pslam_reference_adapter.hpp ../include/pslam_abi.h _ref/libmatch_ref.so ../planarslam_b200/libpslam_b200.so $(SHIMS)
	$(REFCXX) $(REFFLAGS) -std=gnu++17 -DPSLAM_REF_FULL_HEADERS -I ../include -o $@ ref/frame_adapter_driver.cc -L_ref -lmatch_ref -L../planarslam_b200 -lpslam_b200 \
	  $(REFLINK) -Wl,--no-undefined -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../planarslam_b200'
frame-adapter: $(OUT)
	@if [ -d $(REF)/src ] && [ -f ../planarslam_b200/libpslam_b200.so ]; then $(MAKE) --no-print-directory -f ref/frame_adapter.mk _ref/libmatch_ref.so _ref/libframe_adapter_ref.so; \
	else echo "frame adapter test library: prerequisites absent, keeping the prebuilt one"; fi
.PHONY: frame-adapter
