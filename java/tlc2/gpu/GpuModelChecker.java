/*
 * Thin Java driver with tlc2.TLC's argument surface: replaces ModelChecker.doInit/runTLC (the
 * Worker next-state loop, FPSet and StateQueue) by one kmc_run on the GPU.  NOT COMPILED HERE.
 *
 *   java -Djava.library.path=build -cp java tlc2.gpu.GpuModelChecker -config Kip320.cfg -deadlock Kip320
 *
 * The .tla/.cfg pair is lowered ahead of time by `python -m kafka_specification_b200.build`
 * (or by the tlc2-compatible CLI, which does both steps: python -m kafka_specification_b200.tlc2).
 */
package tlc2.gpu;

public final class GpuModelChecker {
    public static void main(String[] args) {
        String config = null, spec = null, modelLib = System.getProperty("kspec.model");
        boolean noDeadlock = false, cont = false, spill = false, setSpill = false;
        int gpus = 1, fpbits = 0;
        String metadir = null, recover = null;
        double checkpointMinutes = -1;
        for (int i = 0; i < args.length; i++) {
            switch (args[i]) {
                case "-config": config = args[++i]; break;
                case "-deadlock": noDeadlock = true; break;
                case "-continue": cont = true; break;
                case "-workers": {                     // N GPUs of this machine behind one context (option "gpus")
                    String w = args[++i];
                    gpus = w.equals("auto") ? 1 : Math.max(1, Integer.parseInt(w));
                    break;
                }
                case "-fpbits": fpbits = Integer.parseInt(args[++i]); break;
                case "-metadir": metadir = args[++i]; break;
                case "-checkpoint": checkpointMinutes = Double.parseDouble(args[++i]); break;
                case "-recover": recover = args[++i]; break;
                case "-spill": spill = true; break;    // extension: old BFS levels move to host memory
                case "-setspill": setSpill = true; break;    // extension: the set's keys move to host memory when its table fills
                default: spec = args[i];
            }
        }
        if (modelLib == null) {
            System.err.println("Error: -Dkspec.model=<libkmc_*.so> is required (AOT-lowered " + spec + " + " + config + ")");
            System.exit(150);
        }
        StringBuilder opts = new StringBuilder("{");
        opts.append("\"continue\": ").append(cont);
        if (noDeadlock) opts.append(", \"check_deadlock\": false");
        if (gpus > 1) opts.append(", \"gpus\": ").append(gpus);
        if (fpbits > 0) opts.append(", \"table_log2\": ").append(fpbits);
        if (spill) opts.append(", \"spill\": true");
        if (setSpill) opts.append(", \"set_spill\": true");
        if (metadir != null) {
            opts.append(", \"checkpoint_dir\": \"").append(metadir).append("\"");
            opts.append(", \"checkpoint_minutes\": ").append(checkpointMinutes < 0 ? 30.0 : checkpointMinutes);
        }
        if (recover != null) opts.append(", \"recover\": \"").append(recover).append("\"");
        opts.append("}");
        long ctx = Native.create(modelLib, opts.toString());
        int rc = Native.run(ctx);
        long[] st = Native.stats(ctx);
        long[] v = Native.violation(ctx);
        int exit = 0;
        if (rc != 0) {
            System.out.println("Error: " + Native.strerror(ctx, rc));
            exit = 1;
        } else if (v != null) {
            System.out.println(v[0] == 2 ? "Error: Deadlock reached." : "Error: Invariant #" + v[1] + " is violated.");
            exit = v[0] == 2 ? 11 : 12;
        } else {
            System.out.println("Model checking completed. No error has been found.");
        }
        System.out.println(st[1] + " states generated, " + st[0] + " distinct states found, " + st[2] + " states left on queue.");
        if (st[8] == 1) System.out.println("The depth of the complete state graph search is " + st[3] + ".");
        Native.destroy(ctx);
        System.exit(exit);
    }
}
