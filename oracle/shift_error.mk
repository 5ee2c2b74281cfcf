# oracle/shift_error.mk -- the reference's test_shifted.c with its DISPLAY_ERROR check switched on.  TEST INFRASTRUCTURE, never
# the product.  It includes oracle/Makefile for its variables and object rules, and adds:
#
#   make -f shift_error.mk shift-error-ref   _ref/* (only when $(REF)/src exists; only binaries land in oracle/_ref/):
#     _ref/ref_test_shifted_error_stock   test_shifted.c -DDISPLAY_ERROR with the reference's own sources on the mini-MPI
#     _ref/ref_test_shifted_error_b200    the same driver, source unchanged, linked against libbicgstab_b200.so (its
#                                         MPI_Allreduce comes from include/compat/mpi.h)
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := shift-error-ref
.PHONY: shift-error-ref

ifneq ($(wildcard $(SRC)/test_shifted.c),)
shift-error-ref: $(OUT)/ref_test_shifted_error_stock $(OUT)/ref_test_shifted_error_b200
else
shift-error-ref:
	@echo "oracle: $(SRC)/test_shifted.c not present -- using prebuilt oracle/_ref if any"
endif

$(OUT)/ref_test_shifted_error_stock: $(SRC)/test_shifted.c $(SRC)/shifted_solver.c $(SRC)/matrix.c $(SRC)/vector.c $(SRC)/mmio.c $(OUT)/mini_mpi.o
	$(CC) $(FAST) $(WARN) $(INC) -DDISPLAY_ERROR -o $@ $^ -lm
$(OUT)/ref_test_shifted_error_b200: $(SRC)/test_shifted.c $(B200LIB)/libbicgstab_b200.so | $(OUT)
	$(CC) -O2 $(WARN) -DDISPLAY_ERROR -I$(abspath $(HERE)../include/compat) -I$(SRC) $(SRC)/test_shifted.c -L$(B200LIB) -lbicgstab_b200 \
	      -Wl,-rpath,'$$ORIGIN/../../mpi-bicgstab_b200' -o $@ -lm
