# ORACLE build (test infrastructure): DDMin with RandomScheduler as the test oracle.  Output:
# oracle/liboracle_random_ddmin.so (git-ignored).  The same sources as liboracle.so (Makefile), with ddmin.c replaced by
# random_ddmin.c, which includes it and adds the random-oracle test, its threaded batch and the minimizer.
CC ?= gcc
CFLAGS ?= -O3 -march=native -fPIC -Wall -Wextra -std=gnu11 -pthread
SRCS := machine.c models.c model_ir.c fuzz.c sts.c dpor.c dpor_frontier.c intmin.c provenance.c random_ddmin.c
liboracle_random_ddmin.so: $(SRCS) ddmin.c machine.h jrandom.h ../include/demi_b200.h ../include/demi_limits.h ../include/demi_model_ir.h
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS)
clean:
	rm -f liboracle_random_ddmin.so
